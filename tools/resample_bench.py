"""The resampler (sab_resample) on 30 minutes of audio: 44.1 kHz stereo -> 48 kHz (the channel mean taken as the kernel
loads) and 48 kHz mono -> 16 kHz, on the engine of the sam-audio-tiny stand-in (the kernel needs no weights).

For each case, with the card's name and power limit read in the same run:
  - kernel time: CUDA events around --iters calls after --warmup, per call (the descriptor upload included);
  - bytes the algorithm needs (every input sample read once, every output written once, fp32) over that time, and its
    share of the H100 SXM data-sheet HBM bandwidth, 3.35 TB/s;
  - torchaudio.functional.resample on the same GPU and the same data, where its dense [new', 1, 2w + orig'] kernel fits
    (mono input: the channel mean in PyTorch first; TF32 convolutions off, so both sides compute in fp32), timed the
    same way, and the largest difference from ours.
Prints one JSON line at the end.  Fails without a GPU.

    python tools/resample_bench.py [--seconds 1800] [--iters 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from stream_bench import card  # noqa: E402  (tools/ is the script's directory)

HBM_BYTES_PER_S = 3.35e12


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def case(eng, orig, new, C, seconds, args):
    from sam_audio_b200.resample import resampled_length
    L = int(orig * seconds)
    g = torch.Generator(device="cuda").manual_seed(orig + C)
    x = 0.1 * torch.randn(C, L, generator=g, device="cuda")
    N = resampled_length(L, orig, new)
    y = torch.empty(N, device="cuda")
    seg = dict(orig_rate=orig, new_rate=new, channels=C, in_=x.data_ptr(), in_channel_stride=L, in_first=0, in_count=L,
               length=L, out=y.data_ptr(), out_first=0, out_count=N)
    ms = timed(lambda: eng.resample([seg]), args.iters, args.warmup)
    nbytes = 4.0 * (C * L + N)
    res = {"orig": orig, "new": new, "channels": C, "input_samples": L, "outputs": N, "ms": ms, "bytes": nbytes,
           "GB_per_s": nbytes / ms / 1e6, "share_of_hbm": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
    try:
        import torchaudio
        mono = x.mean(0) if C > 1 else x[0]
        ta_ms = timed(lambda: torchaudio.functional.resample(mono, orig, new), max(3, args.iters // 4), 1)
        ref = torchaudio.functional.resample(mono, orig, new)
        res.update(torchaudio_ms=ta_ms, torchaudio_max_abs_diff=float((ref - y).abs().max()))
    except (RuntimeError, ImportError) as exc:            # the dense kernel does not fit, or no torchaudio
        res.update(torchaudio_ms=None, torchaudio_error=str(exc)[:200])
    print(f"{orig} -> {new} Hz, C={C}, {seconds:.0f} s: {ms:.3f} ms, {res['GB_per_s']:.0f} GB/s "
          f"({100 * res['share_of_hbm']:.1f}% of 3.35 TB/s); torchaudio {res.get('torchaudio_ms')} ms", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1800.0)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "resample_bench needs a GPU"
    torch.backends.cudnn.allow_tf32 = False
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.model import build_synthetic_model
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    m = build_synthetic_model("sam-audio-tiny", seed=0, device="cuda:0")
    eng = m._ensure_engine()
    cases = [case(eng, 44100, 48000, 2, args.seconds, args), case(eng, 48000, 16000, 1, args.seconds, args)]
    print(json.dumps({"device": name, "power_limit": limit, "seconds": args.seconds, "cases": cases}))


if __name__ == "__main__":
    main()
