"""The int4 / int8 decoder at the 2B and 0.5B widths and with grouped-query heads, bit for bit against the bf16 decoder.

The quantised weight stream rebuilds exactly W = bf16(bf16(q - zero) * scale) in front of the bf16 stream's MMAs, with
the same split plan (gemm_quant.cu), and prefill dequantises each block into the bf16 weights' scratch before the
same row-form GEMMs.  So at any width a quantised engine gives the same bits as the bf16 engine on the dequantised
weights, and that engine's fp64 reference (test_decoder_gpu._Ref) bounds both.  The int8 engines quantise at load
time (quant.quantize_decoder); the int4 engines load a reference-format checkpoint made from that quantisation with
fractional bf16 zero points, so the inner rounding of bf16(bf16(q - zero) * scale) matters.

  * decode step (md_text_decode_step): x, the post-LN output and the whole KV pool are bit-identical; only the new
    token's slots change; layer-1 K/V, x and the post-LN output follow the fp64 reference.  Batches 1, 32 and 130
    (two launches of every weight stream), plus 128 / 129 around the launch boundary at 0.5B.  At 2B and 0.5B the
    [proj | fc2] stream has splits that start on an odd k-block and span several, so they read the scale / zero
    tables at an offset; the grouped-query shape finishes the stream with decode_qkv_finish.
  * prefill (md_text_prefill): x and the pool are bit-identical, and a second prefill after a decode step repeats the
    first (every block is dequantised again into the one shared scratch).
  * BASELINE.json config 5 end to end: the 0.5B preset, int8, batch 128, 256 greedy tokens, streamed and not.
"""
import ctypes
import gc
import math

import pytest
import torch

from test_decoder_gpu import (LAYOUTS, PAGE, _assert_only_rows_changed, _check_against_reference, _config,
                              _decode_positions, _expected_slots, _gather_rows, _kv, _lib, _pool, _Ref, _tables,
                              _write_history)

pytestmark = pytest.mark.gpu

# id: (dim, heads, kv heads, ff)
QSHAPES = {
    "2b": (2048, 32, 32, 8192),
    "0.5b": (1024, 16, 16, 4096),
    "gqa4": (2048, 32, 8, 8192),
}


@pytest.fixture(scope="module")
def engines(request):
    """(name, bits, cfg, quantised engine, bf16 engine on the dequantised weights, bf16 engine on the original
    weights, fp64 reference on the dequantised weights) for a two-layer decoder over the tiny vision tower.  The int4
    engine loads a reference-format checkpoint with fractional zero points."""
    from moondream_b200 import quant, synth
    from moondream_b200.engine import Engine

    name, bits = request.param
    cfg = _config(QSHAPES[name])
    sd = synth.synthetic_state_dict(cfg, 5)
    qt, deq = quant.quantize_decoder(cfg, sd, bits)
    if bits == 8:
        eng_q = Engine(cfg, sd, max_batch=1, kv_pages=1, quantize="int8")        # the tests bring their own KV pools
    else:
        # a reference-format checkpoint whose bf16 zero points are fractional, so that bf16(q - zero) rounds
        g = torch.Generator().manual_seed(len(name))
        for i, blk in enumerate(qt.blocks):
            for key, ql in blk.items():
                ql.zero = (ql.zero + torch.rand(ql.zero.shape, generator=g) - 0.5).bfloat16().float()
                deq[f"text.blocks.{i}.{key}.weight"] = ql.dequantized()
        ck = {k: v for k, v in sd.items() if deq[k] is sd[k]}
        ck.update(quant.reference_checkpoint_entries(cfg, qt))
        eng_q = Engine(cfg, ck, max_batch=1, kv_pages=1)
    assert eng_q.quantized is not None and eng_q.quantized.bits == bits
    eng_d = Engine(cfg, deq, max_batch=1, kv_pages=1)
    eng_b = Engine(cfg, sd, max_batch=1, kv_pages=1)
    yield name, bits, cfg, eng_q, eng_d, eng_b, _Ref(cfg, deq)
    del eng_q, eng_d, eng_b
    gc.collect()
    torch.cuda.empty_cache()


def _cases(extra):
    return [pytest.param((m, bits), x, id=f"{m}-int{bits}-{x}") for m in QSHAPES for bits in (4, 8) for x in extra(m)]


def _same_bits(a, b):
    return torch.equal(a.view(torch.int16), b.view(torch.int16))


def _decode(eng, x0, positions, pool0, bt):
    """md_text_decode_step on copies of x0 and pool0, with a NaN-filled workspace -> (x, normed, pool)"""
    N, lib = _lib()
    B = x0.shape[0]
    x, pool = x0.clone(), pool0.clone()
    normed = torch.full_like(x, float("nan"))
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    bt_dev = bt.cuda()
    kv = _kv(pool, bt_dev)
    ws = torch.full((int(lib.md_text_decode_workspace_bytes(eng.model, B)),), 255, dtype=torch.uint8, device="cuda")
    N.check(lib.md_text_decode_step(eng.model, N.ptr(x), N.ptr(pos), B, ctypes.byref(kv), N.ptr(normed), N.ptr(ws),
                                    N.current_stream()), "md_text_decode_step")
    torch.cuda.synchronize()
    return x, normed, pool


def _prefill(eng, x0, seqs, prefix_len, pool0, bt):
    """md_text_prefill on copies of x0 and pool0, with a NaN-filled workspace -> (x, pool)"""
    N, lib = _lib()
    T = x0.shape[0]
    x, pool = x0.clone(), pool0.clone()
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
    return x, pool


# ------------------------------------------------------------------------------------------------ 1. decode step
@pytest.mark.parametrize("engines,B", _cases(lambda m: (1, 32, 128, 129, 130) if m == "0.5b" else (1, 32, 130)),
                         indirect=["engines"])
def test_quantised_decode_step(engines, B):
    name, bits, cfg, eng_q, eng_d, eng_b, ref = engines
    D, KVH = cfg.text.dim, cfg.text.n_kv_heads
    tag = f"int{bits} decode {name} B={B}"
    positions = _decode_positions(B)
    gen = torch.Generator().manual_seed(B * 5 + bits + len(name))
    gcu = torch.Generator(device="cuda").manual_seed(B * 13 + bits + len(name))
    bt, n_pages = _tables([p + 1 for p in positions], gen)
    pool0 = _pool(2, n_pages, KVH, "nan", gcu)
    hist = _write_history(pool0, bt, positions, gcu)
    x0 = torch.randn(B, D, generator=gcu, device="cuda").bfloat16()

    x, normed, pool = _decode(eng_q, x0, positions, pool0, bt)
    x_d, normed_d, pool_d = _decode(eng_d, x0, positions, pool0, bt)
    for what, a, b in (("x", x, x_d), ("normed_out", normed, normed_d), ("KV pool", pool, pool_d)):
        assert _same_bits(a, b), f"{tag}: {what} differs from the bf16 engine on the dequantised weights"
    del x_d, normed_d, pool_d
    seqs = [(1, p) for p in positions]
    _assert_only_rows_changed(pool0, pool, _expected_slots(pool, bt, seqs))

    rows = torch.cat([_gather_rows(pool, 1, bt, b, [p]) for b, p in enumerate(positions)])
    x_r, n_r, kv_r = ref.run(x0, seqs, hist, 0, rounded=True)
    x_t, n_t, kv_t = ref.run(x0, seqs, hist, 0, rounded=False)
    _check_against_reference(rows[:, 0], kv_r[1][0], kv_t[1][0], f"{tag} layer-1 K")
    _check_against_reference(rows[:, 1], kv_r[1][1], kv_t[1][1], f"{tag} layer-1 V")
    _check_against_reference(x, x_r, x_t, f"{tag} x")
    _check_against_reference(normed, n_r, n_t, f"{tag} normed")

    # the quantised decoder is a different model from the bf16 one, so the bit-equality above is not vacuous
    x_b, _, _ = _decode(eng_b, x0, positions, pool0, bt)
    assert not torch.equal(x_b, x), f"{tag}: the quantised step gives the bf16 weights' output"


# ------------------------------------------------------------------------------------------------ 2. prefill
@pytest.mark.parametrize("engines,layout", _cases(lambda m: ("image_prefix_x2", "seven_chunks", "full_context")),
                         indirect=["engines"])
def test_quantised_prefill(engines, layout):
    name, bits, cfg, eng_q, eng_d, eng_b, ref = engines
    D, KVH = cfg.text.dim, cfg.text.n_kv_heads
    tag = f"int{bits} prefill {name} {layout}"
    seqs, prefix_len = LAYOUTS[layout]
    gen = torch.Generator().manual_seed(len(layout) * 7 + bits + len(name))
    gcu = torch.Generator(device="cuda").manual_seed(len(layout) * 3 + bits + len(name))
    bt, n_pages = _tables([st + n for n, st in seqs], gen)
    pool0 = _pool(2, n_pages, KVH, "big", gcu)
    _write_history(pool0, bt, [st for _, st in seqs], gcu)
    x0 = torch.randn(sum(n for n, _ in seqs), D, generator=gcu, device="cuda").bfloat16()

    x, pool = _prefill(eng_q, x0, seqs, prefix_len, pool0, bt)
    x_d, pool_d = _prefill(eng_d, x0, seqs, prefix_len, pool0, bt)
    assert _same_bits(x, x_d), f"{tag}: x differs from the bf16 engine on the dequantised weights"
    assert _same_bits(pool, pool_d), f"{tag}: the KV pool differs from the bf16 engine on the dequantised weights"
    del x_d, pool_d
    _assert_only_rows_changed(pool0, pool, _expected_slots(pool, bt, seqs))

    # prefill -> decode step -> prefill: the second prefill dequantises every block again and repeats the first
    bt1, n1 = _tables([1], gen)
    _decode(eng_q, x0[:1], [0], _pool(2, n1, KVH, "nan", gcu), bt1)
    x2, pool2 = _prefill(eng_q, x0, seqs, prefix_len, pool0, bt)
    assert _same_bits(x2, x) and _same_bits(pool2, pool), f"{tag}: a prefill after a decode step gives other bits"


# ------------------------------------------------------------------------------------------------ 3. config 5
def test_int8_streaming_decode_0_5b_batch_128():
    """BASELINE.json config 5: Moondream-0.5B with int8 decoder weights, batch 128, 256 greedy tokens without stopping
    at eos, through generate_stream (chunks concatenated) and generate.  Tokens and margins equal the bf16 engine's
    on the dequantised weights.  The two engines run one after the other, each with a KV pool sized to the workload:
    every image's prefix pages plus, per sequence, the pages past the prefix's full ones."""
    from moondream_b200 import config as C, quant, synth
    from moondream_b200.engine import Engine

    cfg = C.moondream_0_5b()
    sd = synth.synthetic_state_dict(cfg, 0)
    _, deq = quant.quantize_decoder(cfg, sd, 8)
    B, T = 128, 256
    imgs = [synth.synthetic_image(60 + i) for i in range(4)]
    prompts = [synth.synthetic_prompt(70 + i, 3 + i % 9, cfg.text.vocab_size) for i in range(B)]
    prefix = cfg.text.prefix_attn
    total = prefix + max(len(p) for p in prompts) + T + 1
    pages = len(imgs) * math.ceil(prefix / PAGE) + B * (math.ceil(total / PAGE) - prefix // PAGE)

    def run(state_dict, quantize):
        eng = Engine(cfg, state_dict, max_batch=B, kv_pages=pages, quantize=quantize)
        encoded = eng.encode_images(imgs)
        prefixes = [encoded[i % len(imgs)] for i in range(B)]
        streamed = torch.cat(list(eng.generate_stream(prefixes, prompts, T, chunk=32, eos_id=-1)), dim=1)
        res = eng.generate(prefixes, prompts, T, stop_on_eos=False)
        assert streamed.shape == (B, T) and torch.equal(streamed, res.tokens[:, :T])
        del eng, encoded, prefixes
        gc.collect()
        torch.cuda.empty_cache()
        return streamed, res.tokens, res.margins

    streamed, tokens, margins = run(sd, "int8")
    streamed_d, tokens_d, margins_d = run(deq, None)
    assert torch.equal(streamed, streamed_d), "generate_stream: the int8 engine's tokens differ"
    assert torch.equal(tokens, tokens_d), "generate: the int8 engine's tokens differ"
    assert torch.equal(margins, margins_d), "generate: the int8 engine's margins differ"
    assert tokens.unique().numel() > 16, "the decode produced almost no distinct tokens"
    print(f"config 5: {B} x {T} tokens equal, {tokens.unique().numel()} distinct; KV pool {pages} pages; "
          f"peak allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
