"""Weight-only quantised decoder weights on the GPU (SURVEY.md §8 row f3; reference layers.py:38-110).

Parity definition (SURVEY.md §8c): the bf16 path on the DEQUANTISED weights W = bf16(bf16(q - zero) * scale).  The
kernels rebuild exactly W and keep the bf16 stream's split plan, so every comparison below is bit-exact:
  * md_dequantize_weights            == quant.dequantize (itself pinned to the reference's dequantize_tensor, CPU tests)
  * md_linear_small_batch_quant      == md_linear_small_batch_bf16 on W
  * Engine(quantize=...) / a reference-format int4 checkpoint == Engine on W: hidden states, KV, tokens, margins
and the oracle (CPU restatement of the reference) on W bounds the whole thing like every other model-level test."""
import pytest
import torch

pytestmark = pytest.mark.gpu


# per-group scale exponents, cycled so that neighbouring groups differ by orders of magnitude; 2^-133 makes the
# scale itself and every product with it fp32-subnormal
EDGE_EXPONENTS = (-20, 4, -7, 0, -133, 2, -14)


def _edges(bits, n_out, K, g):
    """A QuantLinear built directly: int8 bytes over the whole range (-128, -127, 0, 127 at the start of each row), int4
    nibbles 0 and 15 in both halves of a byte, per-group scales 2^e * (1 + u) with e from EDGE_EXPONENTS, and for int4
    fractional zero points in [0, 16), every other group's bf16-valued (a reference checkpoint stores zero_point as
    bf16; the stream layout holds fp32)."""
    from moondream_b200 import quant

    groups = K // 128
    if bits == 4:
        q = torch.randint(0, 16, (n_out, K), generator=g, dtype=torch.uint8)
        q[:, :8] = torch.tensor([0, 15, 15, 0, 0, 0, 15, 15], dtype=torch.uint8)     # bytes 0xf0, 0x0f, 0x00, 0xff
        zero = torch.rand(n_out, groups, generator=g) * 16
        zero[:, 1::2] = zero[:, 1::2].bfloat16().float()
    else:
        q = torch.randint(0, 256, (n_out, K), generator=g, dtype=torch.uint8)
        q[:, :4] = torch.tensor([128, 129, 0, 127], dtype=torch.uint8)                 # -128, -127, 0, 127
        zero = torch.zeros(n_out, groups)                                              # the int8 layout's zero point
    e = torch.tensor(EDGE_EXPONENTS, dtype=torch.float64)
    idx = (torch.arange(n_out).view(-1, 1) + torch.arange(groups).view(1, -1)) % len(EDGE_EXPONENTS)
    scale = (2.0 ** e[idx] * (1 + torch.rand(n_out, groups, generator=g, dtype=torch.float64))).float()
    return quant.QuantLinear(bits, q, scale.contiguous(), zero.contiguous())


def _packed(bits, n_out, K, seed, awkward=False):
    """(QuantLinear, its dequantised bf16 matrix).  awkward: False = quantised from a random matrix; True = int4
    scales perturbed off bf16 and fractional zero points; "edges" = _edges."""
    from moondream_b200 import quant

    g = torch.Generator().manual_seed(seed)
    if awkward == "edges":
        ql = _edges(bits, n_out, K, g)
        return ql, ql.dequantized()
    w = (torch.randn(n_out, K, generator=g) / K ** 0.5).to(torch.bfloat16)
    if bits == 4:
        nib, scale, zero = quant.quantize_weight_int4(w)
        if awkward:
            scale = scale * (1 + torch.rand(scale.shape, generator=g) * 1e-3)
            zero = zero + torch.rand(zero.shape, generator=g) - 0.5
        ql = quant.QuantLinear(4, nib, scale.float().contiguous(), zero.float().contiguous())
    else:
        q8, s8 = quant.quantize_weight_int8(w)
        groups = K // 128
        ql = quant.QuantLinear(8, q8.view(torch.uint8), s8.float().unsqueeze(1).repeat(1, groups).contiguous(),
                               torch.zeros(n_out, groups))
    return ql, ql.dequantized()


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("n_out,K,awkward", [
    (64, 128, False), (100, 256, True), (640, 1024, True), (2048, 2048, False),
    (14336, 2048, True), (2048, 10240, True),                     # the 2B decoder's W1 = [qkv ; fc1], W2 = [proj | fc2]
    (100, 256, "edges"), (14336, 2048, "edges"), (2048, 10240, "edges")])
def test_dequantize_kernel_is_bit_exact(bits, n_out, K, awkward):
    from moondream_b200 import ops

    ql, want = _packed(bits, n_out, K, n_out + K + bits, awkward)
    dev = [t.cuda() for t in (ql.stream_bytes(), ql.scale, ql.zero)]
    out = torch.full((n_out, K + 64), 7.0, device="cuda", dtype=torch.bfloat16)      # row pitch wider than K
    ops.dequantize_weights(bits, *dev, n_out, K, out=out[:, :K])
    torch.cuda.synchronize()
    assert torch.equal(out[:, :K].cpu(), want)
    assert bool((out[:, K:] == 7.0).all())


STREAM_SHAPES = [  # (batch, n_out, K): 2B [qkv;fc1], fc2-like, 0.5B [qkv;fc1] at b128, ragged batch / rows, tiny
    (32, 14336, 2048), (32, 2048, 8192), (128, 7168, 1024), (70, 1000, 512), (5, 640, 128), (64, 4096, 256),
    # GQA-4 [qkv;fc1] (splits of 11 k-blocks start on odd k-blocks), 0.5B [qkv;fc1] past one 128-row launch, and two
    # more plans with odd split starts at multi-k-block splits
    (32, 11264, 2048), (130, 11264, 2048), (129, 7168, 1024), (256, 7168, 1024), (32, 3072, 4096), (16, 7168, 10240)]


def _plan_smallbatch(n_out, K, sms):
    """gemm.cu plan_smallbatch (kb_divisor 0): (tile rows, k-blocks per split, splits)"""
    k_blocks = -(-K // 64)
    best, best_cost = (128, k_blocks, 1), None
    for kb in range(k_blocks, 0, -1):
        splits = -(-k_blocks // kb)
        if splits > 32 or (kb < 4 and k_blocks >= 4):
            break
        for rows in (128, 64):
            waves = -(-(-(-n_out // rows) * splits) // sms)
            cost = waves * rows * kb + splits * n_out * 32 * 8 // (128 * sms)
            if best_cost is None or cost < best_cost:
                best, best_cost = (rows, kb, splits), cost
    return best


def test_stream_shapes_reach_odd_split_starts():
    """A split that starts on an odd k-block and spans more than one k-block reads the quantisation groups at an
    offset (gl = ((kb0 + j) >> 1) - g0 in smallbatch_gemm_kernel).  Whether STREAM_SHAPES reach that case depends on
    the SM count, so the plan is restated here, checked against the library's split count, and the case required."""
    from moondream_b200 import _native as N

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    odd = []
    for n_out, K in dict.fromkeys((n_out, K) for _, n_out, K in STREAM_SHAPES):
        _, kb, splits = _plan_smallbatch(n_out, K, sms)
        got = N.lib().md_linear_small_batch_splits(n_out, K)
        assert got == splits, f"({n_out}, {K}) on {sms} SMs: the library plans {got} splits, the restated " \
                              f"plan_smallbatch {splits}; update _plan_smallbatch"
        if any(s * kb % 2 and min(kb, -(-K // 64) - s * kb) > 1 for s in range(splits)):
            odd.append((n_out, K))
    assert odd, f"on this device ({sms} SMs) no STREAM_SHAPES entry has a split starting on an odd k-block with more " \
                f"than one k-block: add a shape that does"
    print(f"{sms} SMs: odd split starts with > 1 k-block at {odd}")


@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("batch,n_out,K", STREAM_SHAPES)
def test_quantised_stream_equals_bf16_stream_on_dequantised_weights(bits, batch, n_out, K):
    from moondream_b200 import ops

    ql, w = _packed(bits, n_out, K, batch + n_out + K + bits, awkward="edges")
    g = torch.Generator(device="cuda").manual_seed(batch + K)
    x = torch.randn(batch, K, device="cuda", generator=g).bfloat16()
    b = torch.randn(n_out, device="cuda", generator=g).bfloat16()
    res = torch.randn(batch, n_out, device="cuda", generator=g).bfloat16()
    dev = [t.cuda() for t in (ql.stream_bytes(), ql.scale, ql.zero)]
    wd = w.cuda()
    for mode, r in ((0, None), (1, None), (2, res)):
        want = ops.linear_small_batch(x, wd, b, mode, r)
        got = ops.linear_small_batch_quant(bits, x, *dev, n_out, b, mode, r)
        torch.cuda.synchronize()
        assert torch.equal(got, want), f"mode {mode}: {(got.float() - want.float()).abs().max().item()}"
    # and the stream is a Linear: within one bf16 ulp of the fp32 product (accumulation order is the only freedom)
    ref = (x.float() @ wd.float().t() + b.float()).bfloat16().float()
    got = ops.linear_small_batch_quant(bits, x, *dev, n_out, b, 0, None).float()
    assert (got - ref).abs().max().item() <= ref.abs().max().item() * 2.0 ** -7


NEAR_TIE_ULPS = 4.5          # as in tests/test_model_parity_gpu.py


def _check_tokens(got, oracle_gen, what):
    """exact match, or first divergence at a step where the oracle itself is at a near-tie."""
    n = len(oracle_gen.tokens)
    for i in range(n):
        if got[i] != oracle_gen.tokens[i]:
            assert oracle_gen.margin_ulps[i] < NEAR_TIE_ULPS, \
                f"{what}: token {i} differs ({got[i]} vs {oracle_gen.tokens[i]}) at {oracle_gen.margin_ulps[i]:.1f} ulps"
            return i
    return n


@pytest.fixture(scope="module")
def tiny():
    from moondream_b200 import config as C, synth

    cfg = C.tiny()
    return cfg, synth.synthetic_state_dict(cfg, 0)


def _run(eng, cfg, n_tokens=20):
    from moondream_b200 import synth

    imgs = [synth.synthetic_image(40 + i, *hw) for i, hw in enumerate([(378, 378), (500, 700), (378, 378)])]
    prompts = [synth.synthetic_prompt(50 + i, 5 + 2 * i, cfg.text.vocab_size) for i in range(3)]
    prefixes, feats, img_emb, hidden = eng.encode_images(imgs, return_hidden=True)
    kv = [[(k.clone(), v.clone()) for k, v in eng.prefix_kv_tensors(p)] for p in prefixes]
    res = eng.generate(prefixes, prompts, max_tokens=n_tokens)
    torch.cuda.synchronize()
    return imgs, prompts, hidden.clone(), kv, res


@pytest.mark.parametrize("bits", [4, 8])
def test_quantised_engine_equals_bf16_engine_on_dequantised_weights(tiny, bits):
    from moondream_b200 import quant
    from moondream_b200.engine import Engine
    from oracle.moondream_oracle import OracleModel
    cfg, sd = tiny
    qt, deq = quant.quantize_decoder(cfg, sd, bits)
    eng_q = Engine(cfg, sd, max_batch=4, quantize="int4" if bits == 4 else "int8")
    assert eng_q.quantized is not None and eng_q.quantized.bits == bits
    eng_d = Engine(cfg, deq, max_batch=4)
    imgs, prompts, hid_q, kv_q, res_q = _run(eng_q, cfg)
    _, _, hid_d, kv_d, res_d = _run(eng_d, cfg)
    assert torch.equal(hid_q, hid_d)
    for a, b in zip(kv_q, kv_d):
        for (ka, va), (kb, vb) in zip(a, b):
            assert torch.equal(ka, kb) and torch.equal(va, vb)
    assert torch.equal(res_q.tokens, res_d.tokens)
    assert torch.equal(res_q.margins, res_d.margins)
    # the quantised model is a different model from the bf16 one (the comparison above is not vacuous) ...
    eng_b = Engine(cfg, sd, max_batch=4)
    _, _, hid_b, _, _ = _run(eng_b, cfg, n_tokens=1)
    assert not torch.equal(hid_b, hid_q)
    # ... and the oracle on the dequantised weights bounds it like any other model-level test
    orc = OracleModel(cfg, deq)
    exact = 0
    for i in range(3):
        o = orc.generate(orc.encode_image(imgs[i]), prompts[i], 20)
        exact += int(_check_tokens(res_q.tokens[i].tolist(), o, f"int{bits} image {i}") == len(o.tokens))
    assert exact >= 1


def test_reference_format_int4_checkpoint_loads_and_runs(tiny, tmp_path):
    """a state dict with `…weight.packed / .scale / .zero_point` entries (layers.py:58-76) goes through the loader
    and the engine and generates what the bf16 engine generates on the weights `QuantizedLinear.unpack` builds."""
    from moondream_b200 import quant, weights
    from moondream_b200.engine import Engine
    from oracle.moondream_oracle import dequantized_state_dict

    cfg, sd = tiny
    qt, deq = quant.quantize_decoder(cfg, sd, 4)
    ck = {k: v for k, v in sd.items() if deq[k] is sd[k]}
    ck.update(quant.reference_checkpoint_entries(cfg, qt))
    path = str(tmp_path / "int4.pt")
    torch.save(ck, path)
    loaded = weights.load_state_dict_from_file(path, cfg)
    assert quant.is_quantized_checkpoint(loaded)
    eng = Engine(cfg, loaded, max_batch=4)
    assert eng.quantized is not None and eng.quantized.bits == 4
    _, _, hid, _, res = _run(eng, cfg)
    ref_sd = dequantized_state_dict(ck)                       # the oracle's restatement of QuantizedLinear.unpack
    eng_d = Engine(cfg, {k: ref_sd[k] for k in sd}, max_batch=4)
    _, _, hid_d, _, res_d = _run(eng_d, cfg)
    assert torch.equal(hid, hid_d) and torch.equal(res.tokens, res_d.tokens)
