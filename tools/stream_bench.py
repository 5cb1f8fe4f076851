"""Streaming separation (SAMAudio.stream) on the sam-audio-large stand-in: a recording pushed in 1 s chunks through
10 s windows (W = 250 latent frames), the default ODE (midpoint, 16 steps).

Reports, with the card's name and power limit read in the same run:
  - per-push wall time (host clock around push() and a device synchronise): median, 90th percentile and maximum, over
    all pushes and over the pushes that solved a window;
  - the real-time factor: the summed wall time of the pushes over the duration of the audio pushed;
  - the delay from a sample's arrival to its emission, minimum and maximum, for a live source whose chunks arrive in
    real time and a push that starts when its chunk is complete: a sample s emitted by the push of the chunk that ends
    at sample e waited (e - s) / rate + that push's wall time (this holds while the real-time factor is below 1);
  - the engine's workspace_bytes and torch.cuda.max_memory_allocated after 1, 10 and 100 windows.
Prints one JSON line at the end.  Fails without a GPU.

    python tools/stream_bench.py [--model sam-audio-large] [--windows 100] [--push-seconds 1] [--window-seconds 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    name, limit = torch.cuda.get_device_name(0), "unknown"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = out.splitlines()[0] if out else limit
    except Exception:
        pass
    return name, limit


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * (len(xs) - 1) + 0.5))] if xs else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="sam-audio-large")
    ap.add_argument("--windows", type=int, default=100)
    ap.add_argument("--push-seconds", type=float, default=1.0)
    ap.add_argument("--window-seconds", type=float, default=10.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_bench needs a GPU"
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.synthetic import make_state_dict
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    from sam_audio_b200.windows import stream_hop, window_ramp
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    cfg = stand_in_config(args.model)
    m = SAMAudio(cfg, text_encoder=SyntheticTextEncoder())
    m.load_state_dict(make_state_dict(cfg, seed=0, device="cuda"))
    m = m.eval().cuda()
    m._ensure_engine()
    m._state = None
    torch.cuda.empty_cache()

    sr, hop = cfg.audio_codec.sample_rate, cfg.audio_codec.hop_length
    W = int(round(args.window_seconds * sr / hop))
    H = stream_hop(W)
    halo_enc = m._ensure_engine().codec_tiling(False, W)[0]
    frames = (args.windows - 1) * H + W + halo_enc                  # the last push completes window --windows
    push = int(round(args.push_seconds * sr))
    n = -(-frames * hop // push) * push
    gen = torch.Generator(device="cuda").manual_seed(0)
    wav = 0.1 * torch.randn(n, generator=gen, device="cuda")
    s = m.stream("man speaking", window_seconds=args.window_seconds, seed=0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()

    walls, walls_win, delays_min, delays_max, memory = [], [], [], [], {}
    emitted = 0
    t_all = time.perf_counter()
    for e in range(push, n + 1, push):
        before = s.windows_solved
        t0 = time.perf_counter()
        out = s.push(wav[e - push:e])
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        walls.append(dt)
        if s.windows_solved > before:
            walls_win.append(dt)
        k = out.target.numel()
        if k:                                                      # samples [emitted, emitted + k)
            delays_min.append((e - (emitted + k - 1)) / sr + dt)
            delays_max.append((e - emitted) / sr + dt)
            emitted += k
        for w in (1, 10, 100):
            if s.windows_solved >= w and w not in memory:
                memory[w] = {"windows": s.windows_solved, "workspace_bytes": s.workspace_bytes(),
                             "max_memory_allocated": torch.cuda.max_memory_allocated()}
    total_wall = time.perf_counter() - t_all
    t0 = time.perf_counter()
    tail = s.flush()
    torch.cuda.synchronize()
    flush_s = time.perf_counter() - t0
    assert emitted + tail.target.numel() == -(-n // hop) * hop
    audio_s = n / sr
    res = {
        "device": name, "power_limit": limit, "model": args.model, "window_frames": W, "hop_frames": H,
        "ramp_frames": window_ramp(W), "push_seconds": args.push_seconds, "audio_seconds": audio_s,
        "pushes": len(walls), "windows": s.windows_solved,
        "push_ms": {"median": 1e3 * pct(walls, 0.5), "p90": 1e3 * pct(walls, 0.9), "max": 1e3 * max(walls)},
        "push_with_window_ms": {"median": 1e3 * pct(walls_win, 0.5), "p90": 1e3 * pct(walls_win, 0.9),
                                "max": 1e3 * max(walls_win)},
        "flush_ms": 1e3 * flush_s,
        "real_time_factor": sum(walls) / audio_s,
        "real_time_factor_loop": total_wall / audio_s,
        "delay_s": {"min": min(delays_min), "max": max(delays_max)},
        "memory": {str(k): v for k, v in sorted(memory.items())},
    }
    print(f"{args.model}: {len(walls)} pushes of {args.push_seconds} s, W = {W} frames, {s.windows_solved} windows; "
          f"push median {res['push_ms']['median']:.2f} ms (with a window {res['push_with_window_ms']['median']:.1f} ms), "
          f"real-time factor {res['real_time_factor']:.4f}, delay {res['delay_s']['min']:.2f} .. "
          f"{res['delay_s']['max']:.2f} s", flush=True)
    for k, v in sorted(memory.items()):
        print(f"  after {k} windows: workspace {v['workspace_bytes'] / 1e9:.3f} GB, "
              f"allocator peak {v['max_memory_allocated'] / 1e9:.3f} GB", flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
