"""The decoder's fused kernels against an fp64 reference, at the 2B model's widths, with grouped-query heads and over the
whole 2048-token context.

  * prefill: the QKV projection's bias + RoPE + KV-page epilogue (gemm.cu EPI_QKV_ROPE) and the two-layer block;
  * the paged flash attention of the prefill (md_prefill_attention_bf16) and the decode attention
    (md_decode_attention_bf16), with 1 to 16 query heads per KV head;
  * the decode step (md_text_decode_step): the fused decode prologue or decode_qkv_finish, the [proj | fc2] weight
    stream and the residual + LayerNorm epilogue, up to batch 130 (two launches of every weight stream).

Every KV pool is filled with a recorded pattern before a call and compared bit for bit afterwards, so a kernel may only
write its own (layer, page, row) slots.  Each sequence owns its pages in a random permutation; unused block-table
entries point at a trap page.  Rows the prefill may load but not attend to hold large finite values (the flash kernel
multiplies masked keys by zero); the decode kernels never load such rows, so there they hold NaN, as does every
workspace byte before a call.

Reference: text.py:145-158 in fp64 on the GPU, rounded to bf16 where the reference model rounds ("rounded"), and the
same chain without any intermediate rounding ("truth").  Hidden states and layer-1 K/V must lie within REL_TOL of the
rounded reference and no further from the truth than 1.5x the rounded reference's own distance + 2e-3, the rule of
test_model_parity_gpu.py.
"""
import ctypes
import dataclasses
import zlib

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

PAGE = 64
REL_TOL = 3e-2
ATT_TOL = 6e-3
BIG = 2.0 ** 14

# id: (dim, heads, kv heads, ff)
SHAPES = {
    "2b": (2048, 32, 32, 8192),       # the bench's decoder: fused decode path, 256-wide QKV tiles
    "ff512": (1024, 16, 16, 8192),    # 512 fc1 features per head in the fused decode prologue
    "tail": (1152, 18, 18, 2304),     # 128 fc1 features per head; QKV N = 3456 ends half-way into a 256-wide tile
    "gqa4": (2048, 32, 8, 8192),      # decode_qkv_finish, kv_head = head / 4, grouped-query columns of the epilogue
    "mqa": (1024, 16, 1, 4096),       # one KV head: G = 16, QKV N = 1152 (192-wide tiles)
}

# (length, start_pos) of each sequence, prefix_len (-1 = the model's 730-token image prefix)
LAYOUTS = {
    "image_prefix_x2": ([(730, 0), (730, 0)], -1),
    "seven_chunks": ([(1, 730), (5, 731), (63, 767), (64, 1000), (65, 1024), (129, 1300), (200, 1848)], -1),
    "straddles_prefix": ([(100, 700)], -1),
    "causal_only": ([(17, 0), (300, 0)], 0),
    "full_context": ([(2048, 0)], -1),
}
# the flash kernel loads two pages per key tile and clamps the second to the table's last entry when the width is odd
ODD_WIDTH = ([(130, 900), (65, 0)], -1)      # kv_len 1030 and 65: a 17-entry table

POSITIONS = [0, 1, 63, 64, 127, 128, 729, 730, 1023, 1024, 2046, 2047]


def _lib():
    from moondream_b200 import _native as N

    return N, N.lib()


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _bf(t):
    return t.to(torch.bfloat16).to(torch.float64)


def _same(t):
    return t


# ------------------------------------------------------------------------------------------------ KV pools
def _tables(kv_lens, gen):
    """Block tables: sequence s owns ceil(kv_len / 64) pages drawn from a random permutation; page 0 is the trap page
    that every unused entry names.  The width just covers the longest sequence."""
    own = [max(1, -(-n // PAGE)) for n in kv_lens]
    perm = (torch.randperm(sum(own), generator=gen) + 1).tolist()
    bt = torch.zeros(len(kv_lens), max(own), dtype=torch.int32)
    at = 0
    for s, n in enumerate(own):
        bt[s, :n] = torch.tensor(perm[at: at + n], dtype=torch.int32)
        at += n
    return bt, sum(own) + 1


def _slots(bt, s, positions):
    """(page, row) of token positions of sequence s, as device index tensors"""
    positions = torch.as_tensor(positions, dtype=torch.long)
    return bt[s].long()[positions // PAGE].cuda(), (positions % PAGE).cuda()


def _pool(n_layers, n_pages, kvh, fill, gen):
    shape = (n_layers, n_pages, 2, kvh, PAGE, 64)
    if fill == "nan":
        return torch.full(shape, float("nan"), dtype=torch.bfloat16, device="cuda")
    sign = torch.randint(0, 2, shape, generator=gen, device="cuda", dtype=torch.int16)
    return (sign * 2 - 1).to(torch.bfloat16) * BIG


def _write_history(pool, bt, hist_lens, gen):
    """random K/V (N(0, 1), like the projection's outputs) in rows [0, hist_len) of every sequence and layer;
    returns hist[layer][s] = bf16 [hist_len, 2, KVH, 64]"""
    hist = []
    for layer in range(pool.shape[0]):
        per = []
        for s, n in enumerate(hist_lens):
            val = torch.randn(n, 2, pool.shape[3], 64, generator=gen, device="cuda").bfloat16()
            if n:
                pg, rw = _slots(bt, s, range(n))
                pool[layer][pg, :, :, rw, :] = val
            per.append(val)
        hist.append(per)
    return hist


def _kv(pool, bt_dev):
    N, _ = _lib()
    return N.md_kv(pool=pool.data_ptr(), n_pages=pool.shape[1], block_tables=bt_dev.data_ptr(),
                   max_blocks=bt_dev.shape[1], n_layers=pool.shape[0], n_kv_heads=pool.shape[3])


def _assert_only_rows_changed(before, after, expected):
    """every bf16 of the pool outside the expected (layer, page, row) slots keeps its bit pattern"""
    diff = (before.view(torch.int16) != after.view(torch.int16)).any(dim=5).any(dim=3).any(dim=2)   # [L, P, 64]
    stray = diff & ~expected
    assert not bool(stray.any()), f"{int(stray.sum())} KV rows outside the written slots changed, first at " \
                                  f"(layer, page, row) = {tuple(stray.nonzero()[0].tolist())}"


def _expected_slots(pool, bt, seqs):
    """[L, P, 64] mask of the slots a call writes: the rows of every new token, in every layer"""
    mask = torch.zeros(pool.shape[0], pool.shape[1], PAGE, dtype=torch.bool, device="cuda")
    for s, (n, st) in enumerate(seqs):
        pg, rw = _slots(bt, s, range(st, st + n))
        mask[:, pg, rw] = True
    return mask


def _gather_rows(pool, layer, bt, s, positions):
    pg, rw = _slots(bt, s, positions)
    return pool[layer][pg, :, :, rw, :]          # [n, 2, KVH, 64]


# ------------------------------------------------------------------------------------------------ reference
def _rope64(x, pos, table):
    """rope.py:20-48 on [n, heads, 64]: dims (j, j + 16), j < 16, rotate; split-half in, interleaved out"""
    cos, sin = table[pos, :, 0].double().unsqueeze(1), table[pos, :, 1].double().unsqueeze(1)
    re, im = x[..., :16], x[..., 16:32]
    rot = torch.stack((re * cos - im * sin, re * sin + im * cos), dim=-1).flatten(-2)
    return torch.cat([rot, x[..., 32:]], dim=-1)


def _rope_f32(x, pos, table):
    """the same in fp32 mul / mul / sub, which is how the kernels evaluate it (bit-exact)"""
    re, im = x[..., :16].float(), x[..., 16:32].float()
    cos, sin = table[pos, :, 0].unsqueeze(1), table[pos, :, 1].unsqueeze(1)
    rot = torch.stack((re * cos - im * sin, re * sin + im * cos), dim=-1).flatten(-2)
    return torch.cat([rot, x[..., 32:].float()], dim=-1).bfloat16()


def _prefix_mask(qpos, kv_len, prefix_len):
    """moondream.py:138-146: causal, plus a bidirectional block over the first prefix_len positions"""
    kp = torch.arange(kv_len, device=qpos.device).view(1, -1)
    qp = qpos.view(-1, 1)
    return (kp <= qp) | ((kp < prefix_len) & (qp < prefix_len))


def _attend(q, k, v, mask):
    """softmax(q k^T / 8) v in fp64; q [n, H, 64], k / v [m, KVH, 64]; query head h reads KV head h / G"""
    H = q.shape[1]
    g = H // k.shape[1]
    k, v = k.double().repeat_interleave(g, 1), v.double().repeat_interleave(g, 1)
    q = q.double()
    out = torch.empty_like(q)
    for h0 in range(0, H, 8):                    # bounds the [heads, n, m] score tensor
        hs = slice(h0, h0 + 8)
        s = torch.einsum("nhd,mhd->hnm", q[:, hs], k[:, hs]) / 8.0
        p = torch.softmax(s.masked_fill(~mask, float("-inf")), dim=-1)
        out[:, hs] = torch.einsum("hnm,mhd->nhd", p, v[:, hs])
    return out


class _Ref:
    """The decoder block of text.py:145-158 in fp64, with the model's bf16 roundings or without any."""

    def __init__(self, cfg, sd):
        from moondream_b200.engine import rope_table

        t = cfg.text
        self.D, self.H, self.KVH, self.FF = t.dim, t.n_heads, t.n_kv_heads, t.ff_dim
        self.prefix = t.prefix_attn
        get = lambda k: sd[k].to("cuda", torch.float64)
        self.layers = []
        for i in range(t.n_layers):
            p = f"text.blocks.{i}."
            self.layers.append({k: get(p + k) for k in (
                "ln.weight", "ln.bias", "attn.qkv.weight", "attn.qkv.bias", "attn.proj.weight", "attn.proj.bias",
                "mlp.fc1.weight", "mlp.fc1.bias", "mlp.fc2.weight", "mlp.fc2.bias")})
        self.post = (get("text.post_ln.weight"), get("text.post_ln.bias"))
        self.table = rope_table(64, t.max_context).cuda()

    def run(self, x, seqs, hist, prefix_len, rounded):
        """x [T, D] (the bf16 block input); seqs [(length, start)], hist[layer][s] = [start, 2, KVH, 64] rows already in
        the cache.  Returns the block output, the post-LN output and per layer the new (k, v) rows [T, KVH, 64]."""
        r = _bf if rounded else _same
        D, H, KVH = self.D, self.H, self.KVH
        kvw = KVH * 64
        T = x.shape[0]
        pos = torch.cat([torch.arange(st, st + n) for n, st in seqs]).cuda()
        x = x.double()
        kv_new = []
        for li, L in enumerate(self.layers):
            l = r(F.layer_norm(x, (D,), L["ln.weight"], L["ln.bias"], 1e-5))
            qkv = r(l @ L["attn.qkv.weight"].t() + L["attn.qkv.bias"])
            q = r(_rope64(qkv[:, :D].reshape(T, H, 64), pos, self.table))
            k = r(_rope64(qkv[:, D: D + kvw].reshape(T, KVH, 64), pos, self.table))
            v = qkv[:, D + kvw:].reshape(T, KVH, 64)
            kv_new.append((k, v))
            att = torch.empty(T, H, 64, dtype=torch.float64, device="cuda")
            off = 0
            for s, (n, st) in enumerate(seqs):
                old = hist[li][s].double()
                kk = torch.cat([old[:, 0], k[off: off + n]])
                vv = torch.cat([old[:, 1], v[off: off + n]])
                att[off: off + n] = _attend(q[off: off + n], kk, vv, _prefix_mask(pos[off: off + n], st + n, prefix_len))
                off += n
            att = r(att.reshape(T, D))
            a = r(att @ L["attn.proj.weight"].t() + L["attn.proj.bias"])
            h = r(F.gelu(r(l @ L["mlp.fc1.weight"].t() + L["mlp.fc1.bias"]), approximate="tanh"))
            m = r(h @ L["mlp.fc2.weight"].t() + L["mlp.fc2.bias"])
            x = r(r(x + a) + m)
        normed = r(F.layer_norm(x, (D,), self.post[0], self.post[1], 1e-5))
        return x, normed, kv_new


def _check_against_reference(got, rounded, truth, what):
    """REL_TOL against the rounded reference, and no further from the truth than the rounded reference's own
    distance x 1.5 + 2e-3"""
    assert torch.isfinite(got.double()).all(), f"{what}: non-finite values"
    e_ref = rel(got, rounded)
    e_truth, e_own = rel(got, truth), rel(rounded, truth)
    assert e_ref < REL_TOL, f"{what}: rel err {e_ref:.3e} against the rounded reference"
    assert e_truth <= 1.5 * e_own + 2e-3, f"{what}: rel err {e_truth:.3e} against fp64 truth (reference's own {e_own:.3e})"
    print(f"{what}: rel {e_ref:.2e} vs rounded, {e_truth:.2e} vs truth (rounded reference {e_own:.2e})")


# ------------------------------------------------------------------------------------------------ models
def _config(shape):
    """the tiny vision tower in front of a two-layer decoder of shape (dim, heads, kv heads, ff)"""
    from moondream_b200 import config as C

    dim, heads, kvh, ff = shape
    cfg = C.tiny()
    return dataclasses.replace(
        cfg, text=dataclasses.replace(cfg.text, dim=dim, n_heads=heads, n_kv_heads=kvh, ff_dim=ff, n_layers=2,
                                      vocab_size=2048),
        vision=dataclasses.replace(cfg.vision, proj_out_dim=dim), region=dataclasses.replace(cfg.region, dim=dim))


@pytest.fixture(scope="module")
def model(request):
    """Engine over the tiny vision tower and a two-layer decoder of the given shape, plus its fp64 reference"""
    from moondream_b200 import synth
    from moondream_b200.engine import Engine

    cfg = _config(SHAPES[request.param])
    sd = synth.synthetic_state_dict(cfg, 5)
    eng = Engine(cfg, sd, max_batch=1, kv_pages=1)          # the tests bring their own KV pools
    ref = _Ref(cfg, sd)
    yield request.param, cfg, eng, ref
    del eng, ref
    torch.cuda.empty_cache()


def _weight(eng, key):
    from moondream_b200.synth import state_dict_spec

    return eng.weights[[k for k, _, _ in state_dict_spec(eng.cfg)].index(key)]


# ------------------------------------------------------------------------------------------------ 1. prefill
@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("model", list(SHAPES), indirect=True)
def test_prefill_qkv_rope_epilogue(model, layout):
    """md_text_prefill on two layers.  Layer 0's K/V rows equal, bit for bit, md_layernorm_bf16 -> the row-form GEMM
    with a plain bias epilogue -> RoPE in the kernels' fp32 form; nothing else in the pool changes; layer 1's K/V and
    the block output follow the fp64 reference."""
    from moondream_b200 import ops

    N, lib = _lib()
    name, cfg, eng, ref = model
    seqs, prefix_len = LAYOUTS[layout]
    D, KVH = cfg.text.dim, cfg.text.n_kv_heads
    kvw = KVH * 64
    prefix = cfg.text.prefix_attn if prefix_len < 0 else prefix_len
    seed = zlib.crc32(f"{name}/{layout}".encode())
    gen = torch.Generator().manual_seed(seed)
    gcu = torch.Generator(device="cuda").manual_seed(seed + 1)
    bt, n_pages = _tables([st + n for n, st in seqs], gen)
    pool = _pool(2, n_pages, KVH, "big", gcu)
    hist = _write_history(pool, bt, [st for _, st in seqs], gcu)
    before = pool.clone()
    T = sum(n for n, _ in seqs)
    x0 = torch.randn(T, D, generator=gcu, device="cuda").bfloat16()
    x = x0.clone()
    q_off = [0]
    for n, _ in seqs:
        q_off.append(q_off[-1] + n)
    qo = torch.tensor(q_off, dtype=torch.int32, device="cuda")
    sp = torch.tensor([st for _, st in seqs], dtype=torch.int32, device="cuda")
    bt_dev = bt.cuda()
    kv = _kv(pool, bt_dev)
    ws = torch.full((int(lib.md_text_prefill_workspace_bytes(eng.model, T)),), 255, dtype=torch.uint8, device="cuda")
    N.check(lib.md_text_prefill(eng.model, N.ptr(x), T, N.ptr(qo), N.ptr(sp), len(seqs), max(n for n, _ in seqs),
                                prefix_len, ctypes.byref(kv), N.ptr(ws), N.current_stream()), "md_text_prefill")
    torch.cuda.synchronize()
    _assert_only_rows_changed(before, pool, _expected_slots(pool, bt, seqs))

    # layer 0: the same kernels unfused
    ln = torch.empty_like(x0)
    N.check(lib.md_layernorm_bf16(N.ptr(x0), D, N.ptr(_weight(eng, "text.blocks.0.ln.weight")),
                                  N.ptr(_weight(eng, "text.blocks.0.ln.bias")), N.ptr(ln), D, T, D, N.current_stream()))
    qkv = ops.linear(ln, _weight(eng, "text.blocks.0.attn.qkv.weight"), _weight(eng, "text.blocks.0.attn.qkv.bias"))
    pos = torch.cat([torch.arange(st, st + n) for n, st in seqs]).cuda()
    k0 = _rope_f32(qkv[:, D: D + kvw].view(T, KVH, 64), pos, ref.table)
    v0 = qkv[:, D + kvw:].view(T, KVH, 64)
    rows = [torch.cat([_gather_rows(pool, layer, bt, s, range(st, st + n)) for s, (n, st) in enumerate(seqs)])
            for layer in range(2)]
    for what, got, want in (("K", rows[0][:, 0], k0), ("V", rows[0][:, 1], v0)):
        bad = (got.view(torch.int16) != want.view(torch.int16)).any(-1).any(-1)
        assert not bool(bad.any()), f"layer-0 {what}: {int(bad.sum())} of {T} token rows differ, first at token " \
                                    f"{int(bad.nonzero()[0])} (position {int(pos[bad.nonzero()[0]])})"

    # layer 1 and the output against fp64
    x_r, _, kv_r = ref.run(x0, seqs, hist, prefix, rounded=True)
    x_t, _, kv_t = ref.run(x0, seqs, hist, prefix, rounded=False)
    tag = f"prefill {name} {layout}"
    _check_against_reference(rows[1][:, 0], kv_r[1][0], kv_t[1][0], f"{tag} layer-1 K")
    _check_against_reference(rows[1][:, 1], kv_r[1][1], kv_t[1][1], f"{tag} layer-1 V")
    _check_against_reference(x, x_r, x_t, f"{tag} x")


# ------------------------------------------------------------------------------------------------ 2. prefill attention
@pytest.mark.parametrize("layout", list(LAYOUTS) + ["odd_width"])
@pytest.mark.parametrize("G", [1, 4, 16])
def test_prefill_attention(G, layout):
    """md_prefill_attention_bf16 on random q and random cache contents (16 query heads, 16 / G KV heads) against fp64;
    one CTA per work item (impl 4) gives the same bits as the persistent grid; the legacy mma.sync kernel (impl 1,
    multi-head only) meets the same bound."""
    N, lib = _lib()
    seqs, prefix_len = ODD_WIDTH if layout == "odd_width" else LAYOUTS[layout]
    prefix = 730 if prefix_len < 0 else prefix_len
    H, KVH, layer = 16, 16 // G, 1
    gen = torch.Generator().manual_seed(G * 1000 + len(layout))
    gcu = torch.Generator(device="cuda").manual_seed(G * 7 + len(layout))
    kv_lens = [st + n for n, st in seqs]
    bt, n_pages = _tables(kv_lens, gen)
    if layout == "odd_width":
        assert bt.shape[1] % 2 == 1
    pool = _pool(2, n_pages, KVH, "big", gcu)
    cache = _write_history(pool, bt, kv_lens, gcu)[layer]
    before = pool.clone()
    T = sum(n for n, _ in seqs)
    q = torch.randn(T, H * 64, generator=gcu, device="cuda").bfloat16()
    q_off = [0]
    for n, _ in seqs:
        q_off.append(q_off[-1] + n)
    qo = torch.tensor(q_off, dtype=torch.int32, device="cuda")
    sp = torch.tensor([st for _, st in seqs], dtype=torch.int32, device="cuda")
    bt_dev = bt.cuda()
    kv = _kv(pool, bt_dev)
    max_q = max(n for n, _ in seqs)

    def run(impl):
        out = torch.full((T, H * 64), float("nan"), dtype=torch.bfloat16, device="cuda")
        lib.md_debug_attention_impl(impl)
        try:
            N.check(lib.md_prefill_attention_bf16(N.ptr(q), H, T, N.ptr(qo), N.ptr(sp), len(seqs), max_q, prefix,
                                                  ctypes.byref(kv), layer, N.ptr(out), N.current_stream()))
            torch.cuda.synchronize()
        finally:
            lib.md_debug_attention_impl(0)
        return out

    def check(out, what):
        assert torch.isfinite(out.float()).all(), f"{what}: non-finite output"
        for s, (n, st) in enumerate(seqs):
            pos = torch.arange(st, st + n, device="cuda")
            want = _attend(q[q_off[s]: q_off[s + 1]].view(n, H, 64), cache[s][:, 0], cache[s][:, 1],
                           _prefix_mask(pos, st + n, prefix)).reshape(n, H * 64)
            e = rel(out[q_off[s]: q_off[s + 1]], want)
            assert e < ATT_TOL, f"{what}: sequence {s} ({n} tokens from {st}): rel err {e:.3e}"

    out = run(0)
    check(out, "persistent")
    assert torch.equal(run(4), out), "one CTA per work item must give the persistent grid's bits"
    if G == 1:
        check(run(1), "mma.sync")
    _assert_only_rows_changed(before, pool, torch.zeros(2, n_pages, PAGE, dtype=torch.bool, device="cuda"))


# ------------------------------------------------------------------------------------------------ 3. decode attention
def _decode_positions(B):
    """every position of POSITIONS (cycled) for a batch, the last one alone for batch 1, a mixed handful for 7"""
    if B == 1:
        return [2047]
    if B == 7:
        return [2047, 0, 1024, 64, 729, 1, 2046]
    return [POSITIONS[b % len(POSITIONS)] for b in range(B)]


@pytest.mark.parametrize("B", [1, 33, 130])
@pytest.mark.parametrize("G", [1, 2, 4, 8, 16])
def test_decode_attention(G, B):
    """md_decode_attention_bf16 (16 query heads, 16 / G KV heads) against fp64; every row a sequence does not own or
    that lies past its position holds NaN, and the pool is left as it was"""
    N, lib = _lib()
    H, KVH, layer = 16, 16 // G, 1
    gen = torch.Generator().manual_seed(G * 131 + B)
    gcu = torch.Generator(device="cuda").manual_seed(G * 17 + B)
    positions = _decode_positions(B)
    bt, n_pages = _tables([p + 1 for p in positions], gen)
    pool = _pool(2, n_pages, KVH, "nan", gcu)
    cache = _write_history(pool, bt, [p + 1 for p in positions], gcu)[layer]
    before = pool.clone()
    q = torch.randn(B, H * 64, generator=gcu, device="cuda").bfloat16()
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    bt_dev = bt.cuda()
    kv = _kv(pool, bt_dev)
    out = torch.full((B, H * 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    N.check(lib.md_decode_attention_bf16(N.ptr(q), H, N.ptr(pos), B, ctypes.byref(kv), layer, N.ptr(out),
                                         N.current_stream()))
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    _assert_only_rows_changed(before, pool, torch.zeros(2, n_pages, PAGE, dtype=torch.bool, device="cuda"))
    worst = 0.0
    for b, p in enumerate(positions):
        full = torch.ones(1, p + 1, dtype=torch.bool, device="cuda")
        want = _attend(q[b].view(1, H, 64), cache[b][:, 0], cache[b][:, 1], full).reshape(H * 64)
        e = rel(out[b], want)
        assert e < ATT_TOL, f"sequence {b} at position {p}: rel err {e:.3e}"
        worst = max(worst, e)
    print(f"decode attention G={G} B={B}: worst rel err {worst:.2e}")


# ------------------------------------------------------------------------------------------------ 4. decode step
DECODE_CASES = [(m, B) for m in SHAPES for B in (1, 7, 32)] + [("ff512", 130), ("mqa", 130)]


@pytest.mark.parametrize("model,B", DECODE_CASES, indirect=["model"])
def test_decode_step(model, B):
    """md_text_decode_step over two layers with random K/V history: the new K/V rows land at (layer, page(pos),
    pos % 64) and nowhere else, layer 0's within one bf16 ulp of the row's largest magnitude; x and the post-LN output
    follow the fp64 reference"""
    N, lib = _lib()
    name, cfg, eng, ref = model
    D, KVH = cfg.text.dim, cfg.text.n_kv_heads
    positions = _decode_positions(B)
    gen = torch.Generator().manual_seed(B * 3 + len(name))
    gcu = torch.Generator(device="cuda").manual_seed(B * 11 + len(name))
    bt, n_pages = _tables([p + 1 for p in positions], gen)
    pool = _pool(2, n_pages, KVH, "nan", gcu)
    hist = _write_history(pool, bt, positions, gcu)
    before = pool.clone()
    x0 = torch.randn(B, D, generator=gcu, device="cuda").bfloat16()
    x = x0.clone()
    normed = torch.full_like(x, float("nan"))
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    bt_dev = bt.cuda()
    kv = _kv(pool, bt_dev)
    ws = torch.full((int(lib.md_text_decode_workspace_bytes(eng.model, B)),), 255, dtype=torch.uint8, device="cuda")
    N.check(lib.md_text_decode_step(eng.model, N.ptr(x), N.ptr(pos), B, ctypes.byref(kv), N.ptr(normed), N.ptr(ws),
                                    N.current_stream()), "md_text_decode_step")
    torch.cuda.synchronize()
    seqs = [(1, p) for p in positions]
    _assert_only_rows_changed(before, pool, _expected_slots(pool, bt, seqs))
    rows = [torch.cat([_gather_rows(pool, layer, bt, b, [p]) for b, p in enumerate(positions)]) for layer in range(2)]

    x_r, n_r, kv_r = ref.run(x0, seqs, hist, 0, rounded=True)
    x_t, n_t, kv_t = ref.run(x0, seqs, hist, 0, rounded=False)
    for plane, what in ((0, "K"), (1, "V")):
        got, want = rows[0][:, plane].double().reshape(B, -1), kv_r[0][plane].reshape(B, -1)
        assert torch.isfinite(got).all(), f"layer-0 {what}: non-finite"
        err = (got - want).abs().max(dim=1).values
        bound = want.abs().max(dim=1).values * 2.0 ** -7
        bad = err > bound
        assert not bool(bad.any()), f"layer-0 {what}: sequence {int(bad.nonzero()[0])} at position " \
                                    f"{positions[int(bad.nonzero()[0])]} is off by {err.max().item():.3e}"
        frac = (got != want).double().mean().item()
        assert frac < 0.05, f"layer-0 {what}: {frac:.3f} of the elements differ"
    tag = f"decode {name} B={B}"
    _check_against_reference(rows[1][:, 0], kv_r[1][0], kv_t[1][0], f"{tag} layer-1 K")
    _check_against_reference(rows[1][:, 1], kv_r[1][1], kv_t[1][1], f"{tag} layer-1 V")
    _check_against_reference(x, x_r, x_t, f"{tag} x")
    _check_against_reference(normed, n_r, n_t, f"{tag} normed")
