"""Times the decode attention alone at the bench's shape (CUDA events) and prints us per layer and GB/s.

B = 32 sequences at positions 762 ... 826 (the bench's 730-token image prefix + prompt + generated tokens), 32 heads,
a 24-layer pool of the real size with every sequence's pages scattered over it.  One sweep is one
md_decode_attention_bf16 launch per layer; the bulk-copy ring kernel (md_debug_attention_impl 0) and the kernel that
loads K/V into registers (impl 2) alternate in the same process.  The bytes are the algorithm's: sum over sequences of
(pos + 1) x 8 KiB (K and V rows of 32 heads) per layer; the percentage is against the H100 SXM data sheet's 3.35 TB/s.

    python tools/decode_attn_bench.py [OUT.json]     # results on stdout; also to OUT.json if given
"""
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from moondream_b200 import _native as N  # noqa: E402

B, H, LAYERS, PAGE = 32, 32, 24, 64
IMPLS = {"ring": 0, "registers": 2}
ROUNDS, SWEEPS = 7, 20
PEAK_GBS = 3350.0


def main():
    assert torch.cuda.is_available(), "decode_attn_bench.py needs a GPU"
    lib = N.lib()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    card = smi[torch.cuda.current_device()] if smi else torch.cuda.get_device_name()
    positions = [762 + (64 * b) // (B - 1) for b in range(B)]          # 762 ... 826
    own = [(p + 1 + PAGE - 1) // PAGE for p in positions]
    gen = torch.Generator().manual_seed(0)
    perm = (torch.randperm(sum(own), generator=gen) + 1).tolist()
    bt = torch.zeros(B, max(own), dtype=torch.int32)
    at = 0
    for s, n in enumerate(own):
        bt[s, :n] = torch.tensor(perm[at: at + n], dtype=torch.int32)
        at += n
    n_pages = sum(own) + 1
    pool = torch.randn(LAYERS, n_pages, 2, H, PAGE, 64, device="cuda").bfloat16()
    bt_dev = bt.cuda()
    kv = N.md_kv(pool=pool.data_ptr(), n_pages=n_pages, block_tables=bt_dev.data_ptr(), max_blocks=bt.shape[1],
                 n_layers=LAYERS, n_kv_heads=H)
    q = torch.randn(B, H * 64, device="cuda").bfloat16()
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    out = torch.empty(B, H * 64, dtype=torch.bfloat16, device="cuda")
    stream = N.current_stream()
    bytes_layer = sum(p + 1 for p in positions) * H * 2 * 64 * 2

    def sweep():
        for layer in range(LAYERS):
            N.check(lib.md_decode_attention_bf16(N.ptr(q), H, N.ptr(pos), B, ctypes.byref(kv), layer, N.ptr(out),
                                                 stream))

    outs, times = {}, {k: [] for k in IMPLS}
    try:
        for name, impl in IMPLS.items():                                  # warm-up, and the outputs to compare
            lib.md_debug_attention_impl(impl)
            sweep()
            torch.cuda.synchronize()
            outs[name] = out.clone()
        for _ in range(ROUNDS):
            for name, impl in IMPLS.items():
                lib.md_debug_attention_impl(impl)
                sweep()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(SWEEPS):
                    sweep()
                e.record()
                torch.cuda.synchronize()
                times[name].append(s.elapsed_time(e) * 1000.0 / (SWEEPS * LAYERS))
    finally:
        lib.md_debug_attention_impl(0)
    same = torch.equal(outs["ring"], outs["registers"])
    res = {"device": card, "batch": B, "heads": H, "positions": [positions[0], positions[-1]], "layers": LAYERS,
           "bytes_per_layer": bytes_layer, "same_bits": same, "impls": {}}
    print(f"{card}: B={B} H={H} positions {positions[0]}..{positions[-1]}, {bytes_layer / 1e6:.1f} MB of K/V per layer")
    for name in IMPLS:
        us = statistics.median(times[name])
        gbs = bytes_layer / (us * 1e-6) / 1e9
        res["impls"][name] = {"us_per_layer_median": us, "us_per_layer_min": min(times[name]),
                              "us_per_layer_max": max(times[name]), "GBps": gbs, "pct_of_3350": 100 * gbs / PEAK_GBS}
        print(f"{name:9s} {us:7.2f} us/layer (min {min(times[name]):.2f}, max {max(times[name]):.2f})  "
              f"{gbs:7.0f} GB/s = {100 * gbs / PEAK_GBS:5.1f} % of 3.35 TB/s")
    print(f"same bits: {same}")
    if len(sys.argv) > 1:
        json.dump(res, open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
