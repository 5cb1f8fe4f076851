"""Many live streams on one engine (SAMAudio.stream_group) on the sam-audio-large stand-in: S streams pushed 1 s per
tick in lockstep through 10 s windows (W = 250 latent frames), the default ODE (midpoint, 16 steps).  Stream i is
pre-rolled with i * H / S frames of audio before the first timed tick, so the streams' windows spread over the ticks
as those of streams that started at independent times do.

For each S of the sweep, after --warmup ticks (every stream has solved its first window and the buckets in use are
planned and captured), over --ticks timed ticks, with the card's name and power limit read in the same run:
  - tick wall time (host clock around group.push() and a device synchronise): median, 90th percentile, maximum;
  - windows per tick (mean, min, max) and the per-window cost (tick time over the windows it solved, median);
  - the filler share: filler items over all items of the ticks' solves (windows.stream_bucket);
  - plan builds and graph captures during the timed ticks (sab_plan_stats), workspace_bytes and the allocator peak;
  - group.close() of all S streams in one flush tick: its wall time and the plans it built per stream that left;
and the same S streams each run alone through SAMAudio.stream(), pushed round-robin (one round = one push per stream;
skipped once a smaller S already missed real time there, or with --no-solo).  The real-time capacity is the largest S
whose 90th-percentile tick (round) is below the push interval.  With --sample-rate every stream runs at that rate
(SAMAudio.stream(sample_rate=...)): each tick then adds one resampling launch in front of the encode and one after the
decode.  Prints one JSON line at the end.  Fails without a GPU.

    python tools/stream_group_bench.py [--streams 16,32,64,96,128] [--ticks 30] [--warmup 20] [--solo-ticks 20]
                                       [--sample-rate 16000]
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from stream_bench import card, pct  # noqa: E402  (tools/ is the script's directory)

PROMPTS = ["man speaking", "dog barking", "a piano playing softly", "rain on the roof", "a crowd cheering",
           "a car engine", "birds singing in the morning", "a woman singing"]


def stats_ms(xs):
    return {"median": 1e3 * pct(xs, 0.5), "p90": 1e3 * pct(xs, 0.9), "max": 1e3 * max(xs)}


def run(m, S, args, solo: bool):
    """S streams for warmup + ticks ticks; returns the timed ticks' (wall seconds, windows) and the plan counters."""
    from sam_audio_b200.windows import stream_hop
    sr, hop = m.cfg.audio_codec.sample_rate, m.cfg.audio_codec.hop_length
    W = int(round(args.window_seconds * sr / hop))
    H = stream_hop(W)
    rate = args.sample_rate or sr
    push = int(round(args.push_seconds * rate))
    n_ticks = args.warmup + (args.solo_ticks if solo else args.ticks)
    gen = torch.Generator(device="cuda").manual_seed(S)
    pre = [(i * H * hop * rate // sr) // S for i in range(S)]
    wav = 0.1 * torch.randn(S, max(pre) + n_ticks * push, generator=gen, device="cuda")
    eng = m._ensure_engine()
    group = None if solo else m.stream_group(window_seconds=args.window_seconds)
    if solo:
        streams = [m.stream(PROMPTS[i % len(PROMPTS)], window_seconds=args.window_seconds, seed=i,
                            sample_rate=args.sample_rate) for i in range(S)]
    else:
        streams = [group.open(PROMPTS[i % len(PROMPTS)], seed=i, sample_rate=args.sample_rate) for i in range(S)]
    for i, s in enumerate(streams):
        if pre[i]:
            s.push(wav[i, :pre[i]])
    pos = list(pre)
    walls, wins = [], []
    for t in range(n_ticks):
        if t == args.warmup:
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            st0, ws0 = eng.plan_stats(), eng.workspace_bytes()
        before = sum(s.windows_solved for s in streams)
        t0 = time.perf_counter()
        if solo:
            for i, s in enumerate(streams):
                s.push(wav[i, pos[i]:pos[i] + push])
        else:
            group.push({s: wav[i, pos[i]:pos[i] + push] for i, s in enumerate(streams)})
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        for i in range(S):
            pos[i] += push
        if t >= args.warmup:
            walls.append(dt)
            wins.append(sum(s.windows_solved for s in streams) - before)
    st1, ws1 = eng.plan_stats(), eng.workspace_bytes()
    peak = torch.cuda.max_memory_allocated()
    keys = ("dit_plan_builds", "graph_captures", "codec_plan_builds")
    t0 = time.perf_counter()
    if group is None:
        for s in streams:
            s.flush()
    else:
        group.close()                                          # every stream leaves in one flush tick
    torch.cuda.synchronize()
    close_s = time.perf_counter() - t0
    st2 = eng.plan_stats()
    churn = {k: st1[k] - st0[k] for k in keys}
    return walls, wins, churn, {"workspace_bytes_start": ws0, "workspace_bytes_end": ws1,
                                "dit_plans_resident": st1["dit_plans_resident"],
                                "codec_plans_resident": st1["codec_plans_resident"], "max_memory_allocated": peak,
                                "close_ms": 1e3 * close_s, "close_plan_builds_per_stream": {k: (st2[k] - st1[k]) / S
                                                                                            for k in keys},
                                "close_max_memory_allocated": torch.cuda.max_memory_allocated()}


def filler(wins, W):
    from sam_audio_b200.windows import stream_bucket, stream_group_capacity, window_groups, window_rows_budget
    cap = stream_group_capacity(W, window_rows_budget())
    live = total = 0
    for n in wins:
        for g0, g1 in window_groups(n, 1, W, window_rows_budget()):
            live += g1 - g0
            total += len(stream_bucket(g1 - g0, cap))
    return (total - live) / total if total else 0.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="sam-audio-large")
    ap.add_argument("--streams", default="16,32,64,96,128")
    ap.add_argument("--ticks", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--solo-ticks", type=int, default=20)
    ap.add_argument("--no-solo", action="store_true")
    ap.add_argument("--push-seconds", type=float, default=1.0)
    ap.add_argument("--window-seconds", type=float, default=10.0)
    ap.add_argument("--sample-rate", type=int, default=None, help="of every stream (default: the model's rate)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_group_bench needs a GPU"
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.synthetic import make_state_dict
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    from sam_audio_b200.windows import stream_hop
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    cfg = stand_in_config(args.model)
    m = SAMAudio(cfg, text_encoder=SyntheticTextEncoder())
    m.load_state_dict(make_state_dict(cfg, seed=0, device="cuda"))
    m = m.eval().cuda()
    m._ensure_engine()
    m._state = None
    torch.cuda.empty_cache()
    W = int(round(args.window_seconds * cfg.audio_codec.sample_rate / cfg.audio_codec.hop_length))
    interval_ms = 1e3 * args.push_seconds

    sweep, solo_sweep = {}, {}
    solo_done = args.no_solo
    for S in [int(x) for x in args.streams.split(",")]:
        walls, wins, churn, mem = run(m, S, args, solo=False)
        per_win = [w / n for w, n in zip(walls, wins) if n]
        sweep[S] = {"tick_ms": stats_ms(walls), "windows_per_tick": {"mean": sum(wins) / len(wins), "min": min(wins),
                                                                      "max": max(wins)},
                    "ms_per_window": 1e3 * pct(per_win, 0.5) if per_win else None, "filler_share": filler(wins, W),
                    "plan_churn": churn, **mem}
        print(f"group S={S}: tick median {sweep[S]['tick_ms']['median']:.1f} ms, p90 {sweep[S]['tick_ms']['p90']:.1f} "
              f"ms, max {sweep[S]['tick_ms']['max']:.1f} ms; {sweep[S]['windows_per_tick']['mean']:.2f} windows per "
              f"tick, {sweep[S]['ms_per_window']:.1f} ms per window, filler {sweep[S]['filler_share']:.3f}, churn "
              f"{churn}, workspace {mem['workspace_bytes_end'] / 1e9:.2f} GB; close {mem['close_ms']:.0f} ms, plans per "
              f"leave {mem['close_plan_builds_per_stream']}", flush=True)
        if not solo_done:
            walls, wins, _, _ = run(m, S, args, solo=True)
            solo_sweep[S] = {"round_ms": stats_ms(walls), "windows_per_round": sum(wins) / len(wins)}
            print(f"solo  S={S}: round median {solo_sweep[S]['round_ms']['median']:.1f} ms, p90 "
                  f"{solo_sweep[S]['round_ms']['p90']:.1f} ms", flush=True)
            solo_done = solo_sweep[S]["round_ms"]["p90"] >= interval_ms
        if sweep[S]["tick_ms"]["p90"] >= interval_ms:
            break
    cap = max([S for S, v in sweep.items() if v["tick_ms"]["p90"] < interval_ms], default=0)
    solo_cap = max([S for S, v in solo_sweep.items() if v["round_ms"]["p90"] < interval_ms], default=0)
    res = {"device": name, "power_limit": limit, "model": args.model, "window_frames": W, "hop_frames": stream_hop(W),
           "sample_rate": args.sample_rate or cfg.audio_codec.sample_rate, "push_seconds": args.push_seconds,
           "ticks": args.ticks, "warmup": args.warmup,
           "realtime_capacity_streams": cap, "solo_realtime_capacity_streams": solo_cap,
           "solo_capacity_bounded_by_sweep": bool(solo_sweep) and max(solo_sweep) == solo_cap,
           "group": {str(k): v for k, v in sweep.items()}, "solo": {str(k): v for k, v in solo_sweep.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
