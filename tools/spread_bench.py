"""The multichannel stems (sab_spread_channels) on 30 minutes of 48 kHz stereo and of 5.1, and the p90 tick of a stream
group of 64 stereo streams with and without keep_channels.

For each kernel case, with the card's name and power limit read in the same run:
  - kernel time: CUDA events around --iters calls after --warmup, per call (the descriptor upload included);
  - bytes the algorithm needs (T and R and the C channels read once, the 2 C stems written once, fp32) over that time,
    and its share of the H100 SXM data-sheet HBM bandwidth, 3.35 TB/s.
The group case runs 64 streams of 48 kHz stereo on the sam-audio-large stand-in in lockstep 1 s pushes through 10 s
windows, stream i pre-rolled with i * H / S frames of audio as in stream_group_bench.py (so the windows spread over the
ticks), --ticks timed ticks alternating in blocks of 5 between a group with keep_channels and one without, after
--warmup-ticks each (tick wall time: host clock around group.push() and a device synchronise).
Prints one JSON line at the end.  Fails without a GPU.

    python tools/spread_bench.py [--seconds 1800] [--iters 20] [--warmup 3] [--streams 64] [--ticks 40] [--no-group]
"""
import argparse
import json
import os
import sys
import time

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


def kernel_case(model, C, seconds, args):
    S = int(48000 * seconds)
    g = torch.Generator(device="cuda").manual_seed(C)
    t, r = 0.1 * torch.randn(2, S, generator=g, device="cuda")
    x = 0.1 * torch.randn(C, S, generator=g, device="cuda")
    ms = timed(lambda: model.spread_channels(t, r, x), args.iters, args.warmup)
    nbytes = 4.0 * S * (2 + 3 * C)
    res = {"channels": C, "samples": S, "ms": ms, "bytes": nbytes, "GB_per_s": nbytes / ms / 1e6,
           "share_of_hbm": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
    print(f"spread_channels C={C}, {seconds:.0f} s at 48 kHz: {ms:.3f} ms, {res['GB_per_s']:.0f} GB/s "
          f"({100 * res['share_of_hbm']:.1f}% of 3.35 TB/s)", flush=True)
    return res


def group_case(args):
    from sam_audio_b200.model import build_synthetic_model
    from sam_audio_b200.windows import stream_hop
    model = build_synthetic_model("sam-audio-large", seed=0, device="cuda:0", weights_device="cuda:0")
    n = args.streams
    g = torch.Generator(device="cuda").manual_seed(1)
    chunk = 0.1 * torch.randn(2, 48000, generator=g, device="cuda")
    hop = model.cfg.audio_codec.hop_length
    H = stream_hop(int(round(10.0 * 48000 / hop)))
    pre = [(i * H * hop) // n for i in range(n)]
    groups = {}
    for keep in (False, True):
        grp = model.stream_group(window_seconds=10.0)
        streams = [grp.open(f"source {i}", seed=i, keep_channels=keep) for i in range(n)]
        groups[keep] = (grp, streams)
        grp.push({s: chunk[:, :max(1, p)] for s, p in zip(streams, pre)})
        for _ in range(args.warmup_ticks):
            grp.push({s: chunk for s in streams})
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for block in range(args.ticks // 5):
        keep = block % 2 == 1
        grp, streams = groups[keep]
        for _ in range(5):
            t0 = time.perf_counter()
            grp.push({s: chunk for s in streams})
            torch.cuda.synchronize()
            times[keep].append(1e3 * (time.perf_counter() - t0))
    for grp, _ in groups.values():
        grp.close()
    res = {}
    for keep, ts in times.items():
        ts = sorted(ts)
        res["keep_channels" if keep else "mono"] = {"ticks": len(ts), "p50_ms": ts[len(ts) // 2],
                                                    "p90_ms": ts[min(len(ts) - 1, int(0.9 * len(ts)))]}
    print(f"group of {n} stereo streams (sam-audio-large, W = 250, 1 s pushes): p90 tick {res['mono']['p90_ms']:.1f} ms "
          f"mono, {res['keep_channels']['p90_ms']:.1f} ms with keep_channels", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1800.0)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--streams", type=int, default=64)
    ap.add_argument("--ticks", type=int, default=40)
    ap.add_argument("--warmup-ticks", type=int, default=12)
    ap.add_argument("--no-group", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "spread_bench needs a GPU"
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.model import build_synthetic_model
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    m = build_synthetic_model("sam-audio-tiny", seed=0, device="cuda:0")
    cases = [kernel_case(m, 2, args.seconds, args), kernel_case(m, 6, args.seconds, args)]
    del m
    torch.cuda.empty_cache()        # the engine allocates with cudaMalloc: give back the kernel cases' cached blocks
    group = None if args.no_group else group_case(args)
    print(json.dumps({"device": name, "power_limit": limit, "seconds": args.seconds, "kernel": cases, "group": group}))


if __name__ == "__main__":
    main()
