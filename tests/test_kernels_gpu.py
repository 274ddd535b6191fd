"""Kernel-level parity on the GPU: each CUDA kernel against a plain torch fp32 reference of the same op."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _lib():
    from moondream_b200 import _native as N

    return N, N.lib()


@pytest.mark.parametrize("rows,dim", [(1, 1152), (37, 2048), (729 * 2, 1152), (5, 720), (64, 128), (9, 4096)])
def test_layernorm(rows, dim):
    N, lib = _lib()
    g = torch.Generator(device="cuda").manual_seed(rows + dim)
    x = (torch.randn(rows, dim, device="cuda", generator=g) * 3 + 0.5).bfloat16()
    w = (1 + 0.1 * torch.randn(dim, device="cuda", generator=g)).bfloat16()
    b = (0.1 * torch.randn(dim, device="cuda", generator=g)).bfloat16()
    y = torch.empty_like(x)
    N.check(lib.md_layernorm_bf16(N.ptr(x), dim, N.ptr(w), N.ptr(b), N.ptr(y), dim, rows, dim, N.current_stream()))
    ref = F.layer_norm(x.float(), (dim,), w.float(), b.float(), 1e-5).bfloat16()
    assert (y.float() - ref.float()).abs().max().item() <= 2.0 ** -6 * ref.float().abs().max().item()
    assert ((y != ref).float().mean().item()) < 0.02


@pytest.mark.parametrize("impl", [0, 1, 4], ids=["wgmma_persistent", "mma_sync", "wgmma_one_item_per_cta"])
@pytest.mark.parametrize("n_crops,heads", [(1, 16), (3, 2), (2, 10), (5, 16)])
def test_vit_attention(n_crops, heads, impl):
    N, lib = _lib()
    seq, hd = 729, 72
    D = heads * hd
    g = torch.Generator(device="cuda").manual_seed(n_crops * 10 + heads)
    qkv = torch.randn(n_crops * seq, 3 * D, device="cuda", generator=g).bfloat16()
    out = torch.empty(n_crops * seq, D, device="cuda", dtype=torch.bfloat16)
    lib.md_debug_attention_impl(impl)
    try:
        N.check(lib.md_vit_attention_bf16(N.ptr(qkv), n_crops, seq, heads, N.ptr(out), N.current_stream()))
        torch.cuda.synchronize()
    finally:
        lib.md_debug_attention_impl(0)
    q, k, v = [t.view(n_crops, seq, heads, hd).transpose(1, 2).float() for t in qkv.chunk(3, dim=-1)]
    ref = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(n_crops * seq, D)
    assert rel(out, ref) < 6e-3, rel(out, ref)


def _paged_setup(n_seqs, heads, layers, n_pages, max_blocks, seed):
    g = torch.Generator().manual_seed(seed)
    pool = torch.zeros(layers, n_pages, 2, heads, 64, 64, dtype=torch.bfloat16, device="cuda")
    perm = torch.randperm(n_pages, generator=g)[: n_seqs * max_blocks].view(n_seqs, max_blocks).int()
    return pool, perm.cuda()


def _gather_kv(pool, bt, layer, seq, length):
    pages = bt[seq].long()
    blk = pool[layer, pages]                     # [P, 2, H, 64, 64]
    kv = blk.permute(1, 2, 0, 3, 4).reshape(2, blk.shape[2], -1, 64)[:, :, :length]
    return kv[0].float(), kv[1].float()


def _rope_ref(x, table, pos):
    # x [T, H, 64] float; reference semantics (rope.py:20-48): split-half in, interleaved out
    re, im = x[..., :16], x[..., 16:32]
    cos, sin = table[pos, :, 0].unsqueeze(1), table[pos, :, 1].unsqueeze(1)
    o_re = re * cos - im * sin
    o_im = re * sin + im * cos
    rot = torch.stack((o_re, o_im), dim=-1).flatten(-2)
    return torch.cat([rot, x[..., 32:]], dim=-1)


@pytest.mark.parametrize("layer", [0, 1])
@pytest.mark.parametrize("impl", [0, 1, 4], ids=["wgmma_persistent", "mma_sync", "wgmma_one_item_per_cta"])
def test_rope_prefill_decode_attention(impl, layer):
    N, lib = _lib()
    lib.md_debug_attention_impl(impl)
    try:
        _rope_prefill_decode_attention(layer)
    finally:
        lib.md_debug_attention_impl(0)


def _rope_prefill_decode_attention(layer):
    from moondream_b200.engine import rope_table

    N, lib = _lib()
    heads, layers, n_pages, max_blocks, prefix = 4, 2, 64, 16, 730
    D = heads * 64
    lens = [730, 730, 17]
    starts = [0, 0, 730]
    n_seqs = len(lens)
    pool, bt = _paged_setup(n_seqs, heads, layers, n_pages, max_blocks, 1)
    table = rope_table(64, 2048).cuda()
    kv = N.md_kv(pool=pool.data_ptr(), n_pages=n_pages, block_tables=bt.data_ptr(), max_blocks=max_blocks,
                 n_layers=layers)
    g = torch.Generator(device="cuda").manual_seed(3)
    # sequence 2 needs its prefix (positions 0..729) in the cache first: run a 730-token prefill for it
    for (lens_i, starts_i) in (([730, 730, 730], [0, 0, 0]), (lens, starts)):
        T = sum(lens_i)
        qkv = torch.randn(T, 3 * D, device="cuda", generator=g).bfloat16()
        qo = torch.tensor([0] + list(np.cumsum(lens_i)), dtype=torch.int32, device="cuda")
        sp = torch.tensor(starts_i, dtype=torch.int32, device="cuda")
        q_out = torch.empty(T, D, device="cuda", dtype=torch.bfloat16)
        N.check(lib.md_rope_kv_write_bf16(N.ptr(qkv), T, heads, N.ptr(qo), N.ptr(sp), n_seqs, N.ptr(table),
                                          N.ptr(q_out), ctypes.byref(kv), layer, N.current_stream()))
        out = torch.empty(T, D, device="cuda", dtype=torch.bfloat16)
        N.check(lib.md_prefill_attention_bf16(N.ptr(q_out), heads, T, N.ptr(qo), N.ptr(sp), n_seqs, max(lens_i),
                                              prefix, ctypes.byref(kv), layer, N.ptr(out), N.current_stream()))
        torch.cuda.synchronize()
        off = 0
        for s in range(n_seqs):
            L, st = lens_i[s], starts_i[s]
            pos = torch.arange(st, st + L, device="cuda")
            x = qkv[off: off + L].float().view(L, 3, heads, 64)
            q_ref = _rope_ref(x[:, 0], table, pos).bfloat16()
            k_ref = _rope_ref(x[:, 1], table, pos).bfloat16()
            assert torch.equal(q_out[off: off + L].view(L, heads, 64), q_ref), "rope(q) must be bit-exact"
            kc, vc = _gather_kv(pool, bt, layer, s, st + L)
            assert torch.equal(kc[:, st:].transpose(0, 1).bfloat16(), k_ref), "rope(k) in cache must be bit-exact"
            assert torch.equal(vc[:, st:].transpose(0, 1).bfloat16(), x[:, 2].bfloat16())
            # attention reference with the prefix-LM mask (moondream.py:138-146)
            qpos = pos.view(-1, 1)
            kpos = torch.arange(st + L, device="cuda").view(1, -1)
            mask = (kpos <= qpos) | ((kpos < prefix) & (qpos < prefix))
            ref = F.scaled_dot_product_attention(q_ref.float().transpose(0, 1), kc, vc, attn_mask=mask)
            ref = ref.transpose(0, 1).reshape(L, D)
            assert rel(out[off: off + L], ref) < 6e-3, (s, rel(out[off: off + L], ref))
            off += L
    # decode: one new token per sequence
    cur = [730, 730, 747]
    qkv = torch.randn(n_seqs, 3 * D, device="cuda", generator=g).bfloat16()
    pos = torch.tensor(cur, dtype=torch.int32, device="cuda")
    q_out = torch.empty(n_seqs, D, device="cuda", dtype=torch.bfloat16)
    N.check(lib.md_rope_kv_write_bf16(N.ptr(qkv), n_seqs, heads, None, N.ptr(pos), n_seqs, N.ptr(table),
                                      N.ptr(q_out), ctypes.byref(kv), layer, N.current_stream()))
    out = torch.empty(n_seqs, D, device="cuda", dtype=torch.bfloat16)
    N.check(lib.md_decode_attention_bf16(N.ptr(q_out), heads, N.ptr(pos), n_seqs, ctypes.byref(kv), layer,
                                         N.ptr(out), N.current_stream()))
    torch.cuda.synchronize()
    for s in range(n_seqs):
        kc, vc = _gather_kv(pool, bt, layer, s, cur[s] + 1)
        q = q_out[s].float().view(heads, 1, 64)
        ref = F.scaled_dot_product_attention(q, kc, vc).reshape(D)
        assert rel(out[s], ref) < 6e-3, (s, rel(out[s], ref))


@pytest.mark.parametrize("vocab", [2048, 16384])
def test_small_batch_argmax_ties_and_mask(vocab):
    """lm_head + argmax: ties resolve to the lowest index (torch.argmax), mask_id is excluded.
    vocab 16384 exercises the two-stage (sliced) argmax, 2048 the single-stage one."""
    import dataclasses

    from moondream_b200 import config as C, synth
    from moondream_b200.engine import Engine

    cfg = C.tiny()
    cfg = dataclasses.replace(cfg, text=dataclasses.replace(cfg.text, vocab_size=vocab))
    sd = synth.synthetic_state_dict(cfg, 0)
    hi = vocab - 3                                                       # a tie across argmax slices
    sd["text.lm_head.weight"][hi] = sd["text.lm_head.weight"][5]       # rows 5 and hi identical -> tie
    sd["text.lm_head.bias"][hi] = sd["text.lm_head.bias"][5]
    sd["text.lm_head.weight"][7] = sd["text.lm_head.weight"][5]
    sd["text.lm_head.bias"][7] = sd["text.lm_head.bias"][5]
    eng = Engine(cfg, sd, max_batch=4)
    B = 6
    h = torch.randn(B, cfg.text.dim, device="cuda").bfloat16()
    ids = torch.empty(B, dtype=torch.int32, device="cuda")
    logits = torch.empty(B, cfg.text.vocab_size, dtype=torch.bfloat16, device="cuda")
    mar = torch.empty(B, dtype=torch.float32, device="cuda")
    eng.lm_head(h, ids, 1, logits=logits, margins=mar)
    w = {k: v.cuda() for k, v in sd.items() if k.startswith("text.post_ln") or k.startswith("text.lm_head")}
    ln = F.layer_norm(h.float(), (cfg.text.dim,), w["text.post_ln.weight"].float(), w["text.post_ln.bias"].float()).bfloat16()
    ref = (ln.float() @ w["text.lm_head.weight"].float().t() + w["text.lm_head.bias"].float()).bfloat16()
    assert rel(logits, ref) < 1e-2
    assert torch.equal(ids.long(), torch.argmax(logits.float(), dim=-1))
    assert torch.equal(logits[:, 5], logits[:, 7]) and torch.equal(logits[:, 5], logits[:, hi])
    # make the tied rows the winners for one sequence: the lowest index must be returned
    h2 = w["text.lm_head.weight"][5:6].float().repeat(B, 1).bfloat16() * 4
    eng.lm_head(h2, ids, 1, logits=logits, margins=mar)
    assert torch.equal(ids.long(), torch.argmax(logits.float(), dim=-1))
    top2 = torch.topk(logits.float(), 2, dim=-1).values
    assert torch.allclose(mar, top2[:, 0] - top2[:, 1])
    eng.lm_head(h, ids, 1, logits=logits)
    best = ids.clone()
    eng.lm_head(h, ids, 1, mask_id=int(best[0]))
    lg = logits.float().clone()
    lg[:, int(best[0])] = -float("inf")
    assert torch.equal(ids.long(), torch.argmax(lg, dim=-1))


@pytest.mark.parametrize("n_crops", [1, 3])
def test_patchify_is_bit_exact(n_crops):
    """prepare_crops' normalisation + create_patches (vision.py:36-40, 44-61) with the reference's own torch ops."""
    from moondream_b200.engine import pixel_lut

    N, lib = _lib()
    crop, patch, k_pad = 378, 14, 592
    g = torch.Generator().manual_seed(n_crops)
    crops = torch.randint(0, 256, (n_crops, crop, crop, 3), dtype=torch.uint8, generator=g)
    lut = pixel_lut().cuda()
    out = torch.full((n_crops * 729, k_pad), 5.0, dtype=torch.bfloat16, device="cuda")
    N.check(lib.md_patchify_u8(N.ptr(crops.cuda()), n_crops, crop, patch, k_pad, N.ptr(lut), N.ptr(out), N.current_stream()))
    torch.cuda.synchronize()
    # reference: NHWC uint8 -> NCHW bf16, (x / 255 - 0.5) / 0.5, then the reshape / permute of create_patches
    x = crops.permute(0, 3, 1, 2).to(torch.bfloat16).div_(255.0).sub_(0.5).div_(0.5)
    B, C, H, W = x.shape
    P = patch
    ref = x.reshape(B, C, H // P, P, W // P, P).permute(0, 2, 4, 1, 3, 5).reshape(B * (H // P) * (W // P), C * P * P)
    assert torch.equal(out[:, : C * P * P].cpu(), ref)
    assert bool((out[:, C * P * P:] == 0).all())


@pytest.mark.parametrize("tilings", [[(1, 1)], [(2, 2), (1, 1), (3, 3)], [(1, 2), (3, 4), (2, 1)],
                                     [(1, 9), (2, 6), (9, 1)], [(6, 2), (1, 1), (1, 9)]])
@pytest.mark.parametrize("dim", [144, 720, 1152])
def test_stitch_pool_concat_matches_the_reference_ops(dim, tilings):
    """reconstruct_from_crops(patch_size = 1) + adaptive_avg_pool2d + concat (image_crops.py:170-231, vision.py:83-88)
    against the oracle's restatement run with torch CPU bf16 ops: bit-exact (fp32 window sums in row-major order,
    divided by the count, like ATen).  (1, 9) and (9, 1) stitch 27 x 179 and 179 x 27 maps, whose pool windows
    are uneven and overlap; the widths are the tiny, 0.5B and 2B encoders'."""
    import torch.nn.functional as F

    from oracle.moondream_oracle import stitch_crops

    N, lib = _lib()
    g, margin = 27, 4
    n_crops = [1 + th * tw for th, tw in tilings]
    offs = [0]
    for c in n_crops:
        offs.append(offs[-1] + c)
    gen = torch.Generator().manual_seed(len(tilings) * 7 + offs[-1])
    feats = torch.randn(offs[-1] * g * g, dim, generator=gen).to(torch.bfloat16)
    out = torch.empty(len(tilings) * g * g, 2 * dim, dtype=torch.bfloat16, device="cuda")
    d_offs = torch.tensor(offs, dtype=torch.int32, device="cuda")
    d_til = torch.tensor(tilings, dtype=torch.int32, device="cuda")
    N.check(lib.md_stitch_pool_concat_bf16(N.ptr(feats.cuda()), N.ptr(d_offs), N.ptr(d_til), len(tilings), g, margin, dim,
                                           N.ptr(out), N.current_stream()))
    torch.cuda.synchronize()
    got = out.cpu().view(len(tilings), g * g, 2 * dim)
    f = feats.view(offs[-1], g, g, dim)
    for i, til in enumerate(tilings):
        glob = f[offs[i]].reshape(g * g, dim)
        stitched = stitch_crops(f[offs[i] + 1: offs[i + 1]], til, margin)
        pooled = F.adaptive_avg_pool2d(stitched.permute(2, 0, 1), output_size=(g, g)).permute(1, 2, 0).reshape(g * g, dim)
        assert torch.equal(got[i, :, :dim], glob)
        assert torch.equal(got[i, :, dim:], pooled), (til, (got[i, :, dim:].float() - pooled.float()).abs().max().item())
