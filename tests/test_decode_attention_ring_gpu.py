"""The decode attention that streams K/V through a bulk-copy ring (attention.cu decode_attention_ring_kernel) against
fp64 and, bit for bit, against the kernel that loads K/V into registers (md_debug_attention_impl 2), which has the
same work split, lane mapping and arithmetic.

  * context lengths around the half-page stages and the pages (1, 8, 9, 63, 64, 65, ...) mixed in one batch, with
    1, 4 and 16 query heads per KV head: rows past the context inside a loaded page hold NaN; the pool is left as it
    was;
  * the same bits from launch to launch, and eager against CUDA-graph replay;
  * both kernels against fp64 at the bench's shape (32 heads, batch 32, positions 762 ... 826);
  * the fused decode step at the 2B widths, batch 1 / 32 / 130: K / V rows, the fc1 GELU rows, x and the post-LN output
    equal the register-loading kernel's bit for bit;
  * ptxas: no spills, and registers / static shared memory that allow the 8 CTAs per SM the kernel is sized for.

Pools, trap pages and the fp64 reference are test_decoder_gpu.py's.
"""
import ctypes
import dataclasses
import os
import re
import subprocess
import sys

import pytest
import torch

from test_decoder_gpu import (ATT_TOL, PAGE, SHAPES, _assert_only_rows_changed, _attend, _config, _kv, _lib, _pool,
                              _tables, _write_history, rel)

ONE_CTA = 2               # md_debug_attention_impl: the register-loading kernel
CTAS_PER_SM = 8           # attention.cu kDecCtasPerSm
RING_BYTES = 24 * 1024    # attention.cu kDecSmem
LENGTHS = [1, 8, 9, 63, 64, 65, 127, 128, 129, 193, 1025, 2048]


def _attention(lib, N, impl, q, H, pos, B, kv, layer):
    out = torch.full((B, H * 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    lib.md_debug_attention_impl(impl)
    try:
        N.check(lib.md_decode_attention_bf16(N.ptr(q), H, N.ptr(pos), B, ctypes.byref(kv), layer, N.ptr(out),
                                             N.current_stream()))
        torch.cuda.synchronize()
    finally:
        lib.md_debug_attention_impl(0)
    return out


def _setup(H, KVH, kv_lens, seed):
    gen = torch.Generator().manual_seed(seed)
    gcu = torch.Generator(device="cuda").manual_seed(seed + 1)
    bt, n_pages = _tables(kv_lens, gen)
    pool = _pool(2, n_pages, KVH, "nan", gcu)
    cache = _write_history(pool, bt, kv_lens, gcu)[1]
    q = torch.randn(len(kv_lens), H * 64, generator=gcu, device="cuda").bfloat16()
    pos = torch.tensor([n - 1 for n in kv_lens], dtype=torch.int32, device="cuda")
    bt_dev = bt.cuda()
    return pool, bt_dev, cache, q, pos, n_pages


def _check(out, q, cache, kv_lens, H, what):
    assert torch.isfinite(out.float()).all(), f"{what}: non-finite output"
    worst = 0.0
    for b, n in enumerate(kv_lens):
        full = torch.ones(1, n, dtype=torch.bool, device="cuda")
        want = _attend(q[b].view(1, H, 64), cache[b][:, 0], cache[b][:, 1], full).reshape(H * 64)
        e = rel(out[b], want)
        assert e < ATT_TOL, f"{what}: sequence {b} with {n} keys: rel err {e:.3e}"
        worst = max(worst, e)
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("G", [1, 4, 16])
def test_context_lengths(G):
    N, lib = _lib()
    H, KVH = 16, 16 // G
    pool, bt_dev, cache, q, pos, n_pages = _setup(H, KVH, LENGTHS, 97 + G)
    kv = _kv(pool, bt_dev)
    before = pool.clone()
    out = _attention(lib, N, 0, q, H, pos, len(LENGTHS), kv, 1)
    worst = _check(out, q, cache, LENGTHS, H, f"G={G}")
    _assert_only_rows_changed(before, pool, torch.zeros(2, n_pages, PAGE, dtype=torch.bool, device="cuda"))
    assert torch.equal(out, _attention(lib, N, ONE_CTA, q, H, pos, len(LENGTHS), kv, 1)), \
        "the ring kernel must give the bits of the register-loading kernel"
    print(f"G={G}: worst rel err {worst:.2e}")


def _bench_shape():
    return [762 + (64 * b) // 31 + 1 for b in range(32)]     # kv_len: positions 762 ... 826


@pytest.mark.gpu
def test_bits_repeat_and_graph():
    """identical bits over launches and under CUDA-graph replay, at the bench's shape"""
    N, lib = _lib()
    H, B = 32, 32
    kv_lens = _bench_shape()
    pool, bt_dev, cache, q, pos, _ = _setup(H, H, kv_lens, 5)
    kv = _kv(pool, bt_dev)
    first = _attention(lib, N, 0, q, H, pos, B, kv, 1)
    for _ in range(3):
        assert torch.equal(_attention(lib, N, 0, q, H, pos, B, kv, 1), first)
    out = torch.full_like(first, float("nan"))
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            rc = lib.md_decode_attention_bf16(N.ptr(q), H, N.ptr(pos), B, ctypes.byref(kv), 1, N.ptr(out),
                                              ctypes.c_void_p(s.cuda_stream))
    N.check(rc, "md_decode_attention_bf16 under capture")
    for _ in range(2):
        out.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, first), "graph replay must give the eager bits"


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [0, ONE_CTA])
def test_bench_shape_against_fp64(impl):
    N, lib = _lib()
    H = 32
    kv_lens = _bench_shape()
    pool, bt_dev, cache, q, pos, _ = _setup(H, H, kv_lens, 11)
    out = _attention(lib, N, impl, q, H, pos, len(kv_lens), _kv(pool, bt_dev), 1)
    print(f"impl {impl}: worst rel err {_check(out, q, cache, kv_lens, H, f'impl {impl}'):.2e}")


@pytest.fixture(scope="module")
def one_layer_2b():
    """a one-layer decoder at the 2B widths: after a step the workspace still holds that layer's fc1 GELU rows"""
    from moondream_b200 import synth
    from moondream_b200.engine import Engine

    cfg = _config(SHAPES["2b"])
    cfg = dataclasses.replace(cfg, text=dataclasses.replace(cfg.text, n_layers=1))
    eng = Engine(cfg, synth.synthetic_state_dict(cfg, 5), max_batch=1, kv_pages=1)
    yield cfg, eng
    del eng
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 32, 130])
def test_fused_step_bits(one_layer_2b, B):
    N, lib = _lib()
    cfg, eng = one_layer_2b
    D, FF, H = cfg.text.dim, cfg.text.ff_dim, cfg.text.n_heads
    positions = [[2047], None, None][[1, 32, 130].index(B)] or [(37 * b + 762) % 2048 for b in range(B)]
    gen = torch.Generator().manual_seed(B)
    gcu = torch.Generator(device="cuda").manual_seed(B + 1)
    bt, n_pages = _tables([p + 1 for p in positions], gen)
    pool0 = _pool(1, n_pages, H, "nan", gcu)
    _write_history(pool0, bt, positions, gcu)
    x0 = torch.randn(B, D, generator=gcu, device="cuda").bfloat16()
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    bt_dev = bt.cuda()
    ws_bytes = int(lib.md_text_decode_workspace_bytes(eng.model, B))
    xcat_off = 3 * ((B * D * 2 + 255) // 256 * 256)

    def step(impl):
        pool, x = pool0.clone(), x0.clone()
        normed = torch.full_like(x, float("nan"))
        ws = torch.full((ws_bytes,), 255, dtype=torch.uint8, device="cuda")
        kv = _kv(pool, bt_dev)
        lib.md_debug_attention_impl(impl)
        try:
            N.check(lib.md_text_decode_step(eng.model, N.ptr(x), N.ptr(pos), B, ctypes.byref(kv), N.ptr(normed),
                                            N.ptr(ws), N.current_stream()), "md_text_decode_step")
            torch.cuda.synchronize()
        finally:
            lib.md_debug_attention_impl(0)
        hid = ws[xcat_off: xcat_off + B * (D + FF) * 2].view(torch.bfloat16).view(B, D + FF)[:, D:]
        return pool, hid.clone(), x, normed

    ref = step(ONE_CTA)
    got = step(0)
    for what, a, b in zip(("K/V pool", "fc1 GELU rows", "x", "normed"), got, ref):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{what} differs from the register-loading kernel"


def test_ptxas_resources():
    """no spills; registers and static shared memory that let 8 CTAs of 128 threads share an SM with their ring"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    from moondream_b200 import build as Bd

    nvcc = os.environ.get("NVCC", "nvcc")
    flags = [f for f in Bd.NVCC_FLAGS if f != "-shared"]
    res = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-c", "attention.cu", "-o", os.devnull], cwd=Bd.CSRC,
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stderr[-2000:]
    blocks = res.stderr.split("Compiling entry function ")[1:]
    found = 0
    for blk in blocks:
        if "decode_attention_ring_kernel" not in blk.split("'")[1]:
            continue
        found += 1
        regs = int(re.search(r"Used (\d+) registers", blk).group(1))
        smem = int(re.search(r"(\d+) bytes smem", blk).group(1)) if "bytes smem" in blk else 0
        spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", blk)
        assert spill.group(1) == "0" and spill.group(2) == "0", blk
        assert regs * 128 * CTAS_PER_SM <= 65536, f"{regs} registers"
        assert CTAS_PER_SM * (RING_BYTES + smem + 1024) <= 228 * 1024, f"{smem} bytes of static shared memory"
    assert found == 2
