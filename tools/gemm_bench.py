"""Time the DiT linear GEMM shapes in isolation (M = 16 000 rows = sam-audio-large at B = 64) through the
sab_test_gemm seam: bf16 operands, fp32 output, the auto-chosen tile (BN = 256, 2-CTA clusters).  CUDA events over
many back-to-back launches; prints TFLOP/s per shape.  A quick loop for GEMM work; bench.py's per-kernel
`kernels` field (the real fused epilogues inside the full step) stays the figure that counts.

    python tools/gemm_bench.py [--iters 50]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (tag, N, K) of the per-layer DiT linears at d = 2816, ffn hidden = 7552
SHAPES = [("attention.qkv", 8448, 2816), ("attention.wo / cross.wq / cross.wo", 2816, 2816),
          ("ffn.w13", 15104, 2816), ("ffn.w2", 2816, 7552)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--M", type=int, default=16000)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "gemm_bench needs a GPU"
    from sam_audio_b200 import _capi
    lib = _capi.lib()
    M = args.M
    res = {"device": torch.cuda.get_device_name(0), "M": M, "shapes": []}
    for tag, N, K in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(N + K)
        a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
        b = torch.randn(N, K, device="cuda", generator=g).bfloat16()
        c = torch.empty(M, N, device="cuda")

        def run():
            _capi.check(lib.sab_test_gemm(M, N, K, a.data_ptr(), b.data_ptr(), c.data_ptr(), 256, 64, 0,
                                          _capi.stream_ptr()))

        for _ in range(args.warmup):
            run()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.iters):
            run()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.iters
        tflops = 2.0 * M * N * K / (ms * 1e-3) / 1e12
        res["shapes"].append({"tag": tag, "N": N, "K": K, "ms": round(ms, 4), "tflops": round(tflops, 1)})
        print(f"{tag:36s} M={M} N={N:6d} K={K:5d}  {ms:8.3f} ms  {tflops:7.1f} TFLOP/s", flush=True)
        del a, b, c
    print(json.dumps(res))


if __name__ == "__main__":
    main()
