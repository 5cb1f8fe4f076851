"""Offline jobs in the filler slots of a stream group (StreamGroup.submit) on the sam-audio-large stand-in: S live streams
pushed 1 s per tick in lockstep through 10 s windows (W = 250 latent frames), the default ODE (midpoint, 16 steps),
pre-rolled as in tools/stream_group_bench.py so that their windows spread over the ticks.

For each S of the sweep, after --warmup ticks without jobs, the timed ticks alternate in blocks of --block ticks
between ticks with a queue of --jobs recordings of --job-seconds each (submitted before the block, cancelled after it,
outside the timing) and ticks without it, in one run, with the card's name and power limit read in the same run:
  - live tick wall time (host clock around group.push() and a device synchronise), minimum, median, p90 and maximum,
    with and without jobs, and the p90 of each block: the spread of the ticks without jobs is the range of their
    blocks' p90, and the tool reports whether the p90 of the ticks with jobs lies inside it;
  - job windows solved per tick, and job audio seconds per wall-clock second (H frames of final audio per job window,
    over the wall time of the ticks with jobs);
  - the filler share of the ticks' solves (windows.stream_bucket) before jobs take it, and after;
  - plan builds and graph captures during the timed ticks (sab_plan_stats) and the workspace before and after.
Prints one JSON line at the end.  Fails without a GPU.

    python tools/stream_jobs_bench.py [--streams 48,64] [--ticks 60] [--block 5] [--warmup 20] [--jobs 2]
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
from stream_group_bench import PROMPTS, stats_ms  # noqa: E402


def solve_slots(wins, W):
    """(slots, live) of the ticks' solves for the given live windows per tick (the bucket rule)."""
    from sam_audio_b200.windows import stream_bucket, stream_group_capacity, window_groups, window_rows_budget
    cap = stream_group_capacity(W, window_rows_budget())
    live = total = 0
    for n in wins:
        for g0, g1 in window_groups(n, 1, W, window_rows_budget()):
            live += g1 - g0
            total += len(stream_bucket(g1 - g0, cap))
    return total, live


def run(m, S, args):
    from sam_audio_b200.windows import stream_hop
    sr, hop = m.cfg.audio_codec.sample_rate, m.cfg.audio_codec.hop_length
    W = int(round(args.window_seconds * sr / hop))
    H = stream_hop(W)
    push = int(round(args.push_seconds * sr))
    n_ticks = args.warmup + args.ticks
    gen = torch.Generator(device="cuda").manual_seed(S)
    pre = [(i * H * hop) // S for i in range(S)]
    wav = 0.1 * torch.randn(S, max(pre) + n_ticks * push, generator=gen, device="cuda")
    job_wav = 0.1 * torch.randn(args.jobs, int(args.job_seconds * sr), generator=gen, device="cuda")
    eng = m._ensure_engine()
    group = m.stream_group(window_seconds=args.window_seconds)
    streams = [group.open(PROMPTS[i % len(PROMPTS)], seed=i) for i in range(S)]
    for i, s in enumerate(streams):
        if pre[i]:
            s.push(wav[i, :pre[i]])
    pos = list(pre)
    ticks = {True: dict(walls=[], wins=[], job_wins=[], blocks=[]), False: dict(walls=[], wins=[], job_wins=[],
                                                                                blocks=[])}
    jobs = []
    for t in range(n_ticks):
        timed = t >= args.warmup
        with_jobs = timed and ((t - args.warmup) // args.block) % 2 == 0
        if timed and t == args.warmup:
            torch.cuda.synchronize()
            st0, ws0 = eng.plan_stats(), eng.workspace_bytes()
        if with_jobs and not jobs:
            jobs = [group.submit(job_wav[j], PROMPTS[(S + j) % len(PROMPTS)], seed=1000 + j) for j in range(args.jobs)]
        elif not with_jobs and jobs:
            for j in jobs:
                j.cancel()
            jobs = []
        torch.cuda.synchronize()
        before = sum(s.windows_solved for s in streams)
        before_jobs = sum(j.windows_solved for j in jobs)
        t0 = time.perf_counter()
        group.push({s: wav[i, pos[i]:pos[i] + push] for i, s in enumerate(streams)})
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        for i in range(S):
            pos[i] += push
        if timed:
            d = ticks[with_jobs]
            if (t - args.warmup) % args.block == 0:
                d["blocks"].append([])
            d["blocks"][-1].append(dt)
            d["walls"].append(dt)
            d["wins"].append(sum(s.windows_solved for s in streams) - before)
            d["job_wins"].append(sum(j.windows_solved for j in jobs) - before_jobs)
    st1, ws1 = eng.plan_stats(), eng.workspace_bytes()
    for j in jobs:
        j.cancel()
    group.close()
    torch.cuda.synchronize()
    keys = ("dit_plan_builds", "graph_captures", "codec_plan_builds")
    res = {"plan_builds_timed": {k: st1[k] - st0[k] for k in keys}, "workspace_bytes_start": ws0,
           "workspace_bytes_end": ws1}
    for with_jobs, d in ticks.items():
        total, live = solve_slots(d["wins"], W)
        jw = sum(d["job_wins"])
        key = "with_jobs" if with_jobs else "without_jobs"
        res[key] = {"ticks": len(d["walls"]), "tick_ms": dict(stats_ms(d["walls"]), min=1e3 * min(d["walls"])),
                    "block_p90_ms": [1e3 * pct(b, 0.9) for b in d["blocks"]],
                    "live_windows_per_tick": sum(d["wins"]) / len(d["wins"]),
                    "filler_share_before": (total - live) / total if total else 0.0,
                    "filler_share_after": (total - live - jw) / total if total else 0.0,
                    "job_windows_per_tick": jw / len(d["walls"]),
                    "job_audio_s_per_wall_s": jw * H * hop / sr / sum(d["walls"])}
    spread = res["without_jobs"]["block_p90_ms"]
    res["p90_with_jobs_within_spread"] = min(spread) <= res["with_jobs"]["tick_ms"]["p90"] <= max(spread)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="sam-audio-large")
    ap.add_argument("--streams", default="48,64")
    ap.add_argument("--ticks", type=int, default=60)
    ap.add_argument("--block", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--jobs", type=int, default=2)
    ap.add_argument("--job-seconds", type=float, default=600.0)
    ap.add_argument("--push-seconds", type=float, default=1.0)
    ap.add_argument("--window-seconds", type=float, default=10.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "stream_jobs_bench needs a GPU"
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.synthetic import make_state_dict
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    cfg = stand_in_config(args.model)
    m = SAMAudio(cfg, text_encoder=SyntheticTextEncoder())
    m.load_state_dict(make_state_dict(cfg, seed=0, device="cuda"))
    m = m.eval().cuda()
    m._ensure_engine()
    m._state = None
    torch.cuda.empty_cache()
    sweep = {}
    for S in [int(x) for x in args.streams.split(",")]:
        r = sweep[S] = run(m, S, args)
        for key in ("without_jobs", "with_jobs"):
            v = r[key]
            print(f"S={S} {key}: tick min {v['tick_ms']['min']:.1f} ms, median {v['tick_ms']['median']:.1f} ms, p90 "
                  f"{v['tick_ms']['p90']:.1f} ms, max {v['tick_ms']['max']:.1f} ms, block p90 "
                  f"{[round(x, 1) for x in v['block_p90_ms']]}, "
                  f"{v['live_windows_per_tick']:.2f} live windows per tick, {v['job_windows_per_tick']:.2f} job "
                  f"windows per tick, {v['job_audio_s_per_wall_s']:.2f} job audio s per wall s, filler "
                  f"{v['filler_share_before']:.3f} -> {v['filler_share_after']:.3f}", flush=True)
        print(f"S={S}: p90 with jobs within the spread of block p90s without: {r['p90_with_jobs_within_spread']}; "
              f"plan builds in timed ticks {r['plan_builds_timed']}, workspace {r['workspace_bytes_start']} -> "
              f"{r['workspace_bytes_end']}", flush=True)
    print(json.dumps({"device": name, "power_limit": limit, "model": args.model, "window_seconds": args.window_seconds,
                      "push_seconds": args.push_seconds, "jobs": args.jobs, "job_seconds": args.job_seconds,
                      "block": args.block, "sweep": {str(k): v for k, v in sweep.items()}}))


if __name__ == "__main__":
    main()
