"""The row-form GEMM's wide column tiles (BN = 192 / 256) give the same bits as 128-wide tiles (md_debug_gemm bit 8):
the K order of every accumulator is the same, only the wgmma instruction's N differs."""
import dataclasses

import pytest
import torch

pytestmark = pytest.mark.gpu

FORCE_128 = 256          # md_debug_gemm bit 8

# (N, K) of the 2B model's row-form layers: ViT qkv / proj / fc1 / fc2, projection fc1 / fc2, prefill qkv / proj / fc1
# (prefill fc2 is the projection's fc2 shape)
SHAPES = [(3456, 1152), (1152, 1152), (4304, 1152), (1152, 4304), (8192, 2304), (2048, 8192), (6144, 2048),
          (2048, 2048), (8192, 2048)]


def _both(fn):
    from moondream_b200 import _native as N_

    lib = N_.lib()
    try:
        lib.md_debug_gemm(FORCE_128)
        narrow = fn()
        lib.md_debug_gemm(0)
        wide = fn()
    finally:
        lib.md_debug_gemm(0)
    torch.cuda.synchronize()
    return wide, narrow


@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_wide_tiles_equal_128(N, K, mode):
    from moondream_b200 import ops

    M = 1000                 # 7 full row tiles and a 104-row tail
    g = torch.Generator(device="cuda").manual_seed(N + K + mode)
    x = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g).bfloat16()
    res = torch.randn(M, N, device="cuda", generator=g).bfloat16() if mode == 2 else None
    wide, narrow = _both(lambda: ops.linear(x, w, b, epilogue=mode, residual=res))
    assert torch.isfinite(wide.float()).all()
    assert torch.equal(wide, narrow), (wide.float() - narrow.float()).abs().max().item()


def test_wide_tiles_posemb_broadcast_and_remap():
    from moondream_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    B, T, K, N = 3, 729, 1152, 1152
    x = torch.randn(B * T, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / K ** 0.5).bfloat16()
    b = torch.randn(N, device="cuda", generator=g).bfloat16()
    pos = torch.randn(T, N, device="cuda", generator=g).bfloat16()
    wide, narrow = _both(lambda: ops.linear(x, w, b, epilogue=2, residual=pos, res_mod=T))
    assert torch.equal(wide, narrow)

    def remapped():
        out = torch.zeros(B * (T + 1), N, device="cuda", dtype=torch.bfloat16)
        return ops.linear(x, w, b, epilogue=0, out=out, remap=(T, T + 1, 1))

    wide, narrow = _both(remapped)
    assert torch.equal(wide, narrow)
    assert wide.view(B, T + 1, N)[:, 0].abs().max().item() == 0


def test_wide_tiles_2b_encode_and_prefill():
    """ViT, projection and the 730-token image prefill of two images at the 2B model's widths (two decoder blocks):
    features, hidden states and every layer's K / V, which covers the QKV + RoPE + KV-page epilogue at 3 - 4 heads per
    column tile."""
    from moondream_b200 import config as C, synth
    from moondream_b200.engine import Engine

    cfg = C.moondream_2b()
    cfg = C.replace(cfg, text=dataclasses.replace(cfg.text, n_layers=2))
    eng = Engine(cfg, synth.synthetic_state_dict(cfg, 3), max_batch=2, kv_pages=64)
    imgs = [synth.synthetic_image(60 + i, 378, 378) for i in range(2)]

    def run():
        prefixes, feats, emb, hidden = eng.encode_images(imgs, return_hidden=True)
        kv = [t for p in prefixes for layer in eng.prefix_kv_tensors(p) for t in layer]
        return [feats.clone(), emb.clone(), hidden.clone()] + kv

    wide, narrow = _both(run)
    assert len(wide) == 3 + 2 * 2 * cfg.text.n_layers
    for i, (a, b) in enumerate(zip(wide, narrow)):
        assert torch.isfinite(a.float()).all(), i
        assert torch.equal(a, b), (i, (a.float() - b.float()).abs().max().item())
