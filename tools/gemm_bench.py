"""Times the wgmma GEMMs on the bench workload's shapes (CUDA events) and prints TFLOP/s / GB/s.

Row form: the 2B model's layers at the M of `bench.py` (64 crops x 729 ViT rows, 32 x 729 projection rows, 32 x (730 +
32) rows of the one-pass image + prompt prefill), each with its epilogue mode.  The prefill QKV layer runs in mode 0
(bias only) as a stand-in for its RoPE + KV-page epilogue.  Every shape is timed with the planned column tile and with
128-wide tiles (md_debug_gemm bit 8), alternating, in the same process; a build without bit 8 times the same plan twice.

    python tools/gemm_bench.py [OUT.json]       # one line per shape on stdout; all rows to OUT.json if given
"""
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from moondream_b200 import _native as N_, ops  # noqa: E402

ROWFORM = [  # name, M, N, K, epilogue mode (0 bias, 1 bias + GELU, 2 bias + residual)
    ("vit_qkv", 46656, 3456, 1152, 0), ("vit_proj", 46656, 1152, 1152, 2), ("vit_fc1", 46656, 4304, 1152, 1),
    ("vit_fc2", 46656, 1152, 4304, 2), ("proj_fc1", 23328, 8192, 2304, 1), ("proj_fc2", 23328, 2048, 8192, 0),
    ("prefill_qkv", 24384, 6144, 2048, 0), ("prefill_proj", 24384, 2048, 2048, 2), ("prefill_fc1", 24384, 8192, 2048, 1),
    ("prefill_fc2", 24384, 2048, 8192, 2),
]
FORCE_128 = 256
ROUNDS = 5


def timeit(fn, iters=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(iters):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def main():
    out = []
    lib = N_.lib()
    dev = torch.cuda.get_device_properties(0)
    for (name, M, N, K, mode) in ROWFORM:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") / K ** 0.5).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        r = torch.randn(M, N, device="cuda").bfloat16() if mode == 2 else None
        y = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        fl = 2 * M * N * K / 1e9
        iters = max(10, int(2e4 / fl))          # ~40 ms of work per sample at 500 TFLOP/s
        ms = {"planned": [], "bn128": []}
        try:
            for _ in range(ROUNDS):
                for key, flags in (("planned", 0), ("bn128", FORCE_128)):
                    lib.md_debug_gemm(flags)
                    ms[key].append(timeit(lambda: ops.linear(x, w, b, epilogue=mode, residual=r, out=y), iters=iters))
        finally:
            lib.md_debug_gemm(0)
        ms_t = timeit(lambda: torch.nn.functional.linear(x, w, b), iters=iters)
        row = {"shape": name, "M": M, "N": N, "K": K, "mode": mode}
        for key, v in ms.items():
            row[key + "_tflops"] = fl / statistics.median(v)
            row[key + "_tflops_all"] = [round(fl / t, 1) for t in v]
        row["torch_linear_tflops"] = fl / ms_t
        out.append(row)
        print(row, flush=True)
        del x, w, b, r, y
    for (B, N, K) in [(32, 6144, 2048), (32, 2048, 2048), (32, 8192, 2048), (32, 2048, 8192),
                      (32, 51200, 2048), (128, 3072, 1024)]:
        x = torch.randn(B, K, device="cuda").bfloat16()
        w = torch.randn(N, K, device="cuda").bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        y = torch.empty(B, N, device="cuda", dtype=torch.bfloat16)
        ws = torch.empty(16 * B * N, device="cuda", dtype=torch.float32)
        ms = timeit(lambda: ops.linear_small_batch(x, w, b, out=y, workspace=ws), iters=50)
        ms_t = timeit(lambda: torch.nn.functional.linear(x, w, b), iters=50)
        out.append({"B": B, "N": N, "K": K, "ms": ms, "gbs": N * K * 2 / ms / 1e6,
                    "torch_ms": ms_t, "torch_gbs": N * K * 2 / ms_t / 1e6})
        print(out[-1], flush=True)
    if len(sys.argv) > 1:
        json.dump({"device": dev.name, "rows": out}, open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
