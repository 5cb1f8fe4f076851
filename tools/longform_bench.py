"""Long-form (T > 256 latent frames) self-attention on the sam-audio-large stand-in, two measurements in one run:

  1. kernels alone, through the C-ABI seams, CUDA events over many launches: the wgmma streaming kernel
     (attention_stream_tc.cuh; bounded and exact softmax) against the mma.sync streaming kernel (attention.cuh) on the
     same shapes, T in {750, 3000, 7500} (30 s, 2 min, 5 min), 22 heads, items chosen so the grid fills the card
     several times over;
  2. one midpoint ODE step (two DiT evaluations, every kernel of the layer stack) of one clip of 30 s and of 5 min,
     default engine against an engine planned under SAB_NO_TC_ATTENTION=1, alternated, every shape warmed up;
  3. separate() end to end on the default engine for each --clips length (default one 5 min clip: codec encode in time
     tiles, 32 evaluations, codec decode in time tiles; past the 400 s position table the DiT runs windowed), host clock
     around a synchronised call, with the real-time factor, the window and group counts, the engine's workspace_bytes
     afterwards and the tile lengths the codec chose.
With --only-separate: the window blend kernel alone (CUDA events; GB/s against 3.35 TB/s), the DiT plan of one window
group at the default row budget, and step 3.

Every timing window is stretched to at least --min-window seconds of GPU work; a row quotes the median of the rounds and
their range.  The kernel rows go through the test seams, which encode three TMA descriptors on the host per call: for
the shortest kernel (T = 750) the host may not keep the GPU busy, and the row is then a lower bound on the kernel's rate.

Achieved TFLOP/s counts 4 * T^2 * 128 per (item, head).  The floor is the larger of FLOPs / 989 TFLOP/s (H100 SXM data
sheet, dense bf16, 700 W) and q|k|v|o once / 3.35 TB/s; the line says which of the two it is.  Prints the card name and
its power limit, and one JSON line at the end.  Fails without a GPU.

    python tools/longform_bench.py [--min-window 0.25] [--model sam-audio-large] [--clips 300,600,1800] [--only-separate]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BF16 = 989e12
PEAK_HBM = 3.35e12
LOG2E = 1.4426950408889634


def card():
    name, limit = torch.cuda.get_device_name(0), "unknown"
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = out.splitlines()[0] if out else limit
    except Exception:
        pass
    return name, limit


def timed(fn, warmup, iters, min_window_s):
    """ms per call over a window of at least min_window_s (the count is scaled up from a first window of `iters`)."""
    for _ in range(warmup):
        fn()
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
        if ms >= min_window_s * 1e3 * 0.9:
            return ms / iters
        iters = int(iters * max(1.5, min_window_s * 1e3 / max(ms, 1e-3))) + 1


def summary(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2], xs[0], xs[-1]


def bench_kernels(args, res):
    from sam_audio_b200 import _capi
    lib = _capi.lib()
    heads = 22
    for T, items in ((750, 4), (3000, 2), (7500, 1)):
        g = torch.Generator(device="cuda").manual_seed(T)
        q, k, v = (torch.randn(items * T, heads * 128, device="cuda", generator=g).bfloat16() for _ in range(3))
        qs = (q.float() * (LOG2E / 128 ** 0.5)).bfloat16()       # as the engine's QKV epilogue leaves q
        mask = torch.ones(items, T, dtype=torch.uint8, device="cuda")
        o = torch.empty_like(q)
        flops = 4.0 * items * heads * T * T * 128
        nbytes = 4.0 * items * T * heads * 128 * 2
        t_fl, t_by = flops / PEAK_BF16, nbytes / PEAK_HBM
        arms = {
            "stream_tc.bounded": lambda: _capi.check(lib.sab_test_attention_stream(
                items, heads, T, qs.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr(), o.data_ptr(), 0.0, -1,
                _capi.stream_ptr())),
            "stream_tc.exact": lambda: _capi.check(lib.sab_test_attention_stream(
                items, heads, T, q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr(), o.data_ptr(), -1.0, -1,
                _capi.stream_ptr())),
            "attention_kernel": lambda: _capi.check(lib.sab_test_attention(
                items, heads, T, T, q.data_ptr(), k.data_ptr(), v.data_ptr(), mask.data_ptr(), o.data_ptr(),
                _capi.stream_ptr())),
        }
        ms = {name: [] for name in arms}
        for _ in range(args.rounds):                             # alternate the arms
            for name, fn in arms.items():
                ms[name].append(timed(fn, args.warmup, args.iters, args.min_window))
        for name, xs in ms.items():
            med, lo, hi = summary(xs)
            row = {"kernel": name, "T": T, "items": items, "heads": heads, "ms_median": round(med, 4),
                   "ms_range": [round(lo, 4), round(hi, 4)], "tflops": round(flops / (med * 1e-3) / 1e12, 1),
                   "bound": "compute" if t_fl >= t_by else "memory",
                   "share_of_floor": round(max(t_fl, t_by) / (med * 1e-3), 3)}
            res["kernels"].append(row)
            print(f"T={T:5d} items={items} heads={heads} {name:18s} median {med:9.4f} ms (range {lo:.4f} .. {hi:.4f}) "
                  f"{row['tflops']:7.1f} TFLOP/s  {row['bound']}-bound floor, share {row['share_of_floor']:.3f}", flush=True)
        del q, k, v, qs, o


@contextlib.contextmanager
def env(name, on):
    """`name` set to 1 (on) or unset (off) inside the block; the caller's own setting is restored afterwards."""
    saved = os.environ.pop(name, None)
    if on:
        os.environ[name] = "1"
    try:
        yield
    finally:
        os.environ.pop(name, None)
        if saved is not None:
            os.environ[name] = saved


def bench_steps(args, res):
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.synthetic import make_state_dict
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    cfg = stand_in_config(args.model)
    sd = make_state_dict(cfg, seed=0, device="cuda")
    models = {}
    for arm, no_tc in (("default", False), ("SAB_NO_TC_ATTENTION=1", True)):
        m = SAMAudio(cfg, text_encoder=SyntheticTextEncoder())
        m.load_state_dict(sd)
        m = m.eval().cuda()
        with env("SAB_NO_TC_ATTENTION", no_tc):
            m._ensure_engine()
        m._state = None
        models[arm] = (m, no_tc)
    del sd
    torch.cuda.empty_cache()
    for seconds, T in ((30, 750), (300, 7500)):
        g = torch.Generator(device="cuda").manual_seed(T)
        f = torch.randn(1, T, 128, device="cuda", generator=g)
        feats = torch.cat([f, f], 2)
        text = torch.randn(1, 4, 768, device="cuda", generator=g)
        ids = torch.tensor([[0, 3]], device="cuda")
        al = torch.zeros(1, T, dtype=torch.long, device="cuda")
        y0 = torch.randn(1, T, 256, device="cuda", generator=g)
        out = torch.empty_like(y0)
        ms = {arm: [] for arm in models}
        outs = {}
        for _ in range(args.rounds):
            for arm, (m, no_tc) in models.items():
                # the plan of a shape is built when it is first prepared: the switch has to be set around that
                with env("SAB_NO_TC_ATTENTION", no_tc):
                    m._install_conditioning(feats, text, None, None, ids, al, None)
                    eng = m._ensure_engine()
                    ms[arm].append(timed(lambda: eng.solve(y0, 1, out), 2, 5, args.min_window))
                outs[arm] = out.clone()
        a, b = outs["default"].double(), outs["SAB_NO_TC_ATTENTION=1"].double()
        diff = float((a - b).norm() / b.norm())
        for arm, xs in ms.items():
            med, lo, hi = summary(xs)
            row = {"arm": arm, "clip_s": seconds, "T": T, "ode_step_ms_median": round(med, 3),
                   "ms_range": [round(lo, 3), round(hi, 3)], "workspace_bytes": models[arm][0]._ensure_engine().workspace_bytes()}
            res["steps"].append(row)
            print(f"{seconds:4d} s clip (T={T}) one midpoint step, {arm:22s} median {med:10.3f} ms (range {lo:.3f} .. {hi:.3f})  "
                  f"workspace {row['workspace_bytes'] / 1e9:.2f} GB", flush=True)
        res["steps"].append({"clip_s": seconds, "arms_rel_l2": diff})
        print(f"{seconds:4d} s clip: the two arms' step outputs differ by rel-L2 {diff:.2e}", flush=True)
    del models["SAB_NO_TC_ATTENTION=1"]
    torch.cuda.empty_cache()
    bench_separate(args, res, models["default"][0], cfg)


def bench_separate(args, res, model, cfg):
    """separate() end to end for each --clips length, host clock around a synchronised call.  Recordings longer than the
    position table (transformer.max_positions frames, 400 s at the default 10 000) run windowed: the window and group
    counts are reported with the times."""
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_noise
    from sam_audio_b200.windows import window_groups, window_layout, window_rows_budget
    hop, sr = cfg.audio_codec.hop_length, cfg.audio_codec.sample_rate
    Tw = cfg.transformer.max_positions
    proc = SAMAudioProcessor(hop, sr)
    eng = model._ensure_engine()
    res["separate"] = []
    for seconds in args.clips:
        T = seconds * sr // hop
        aud = [synthetic_clip(11, seconds * sr)]
        noise = synthetic_noise(1, T).cuda()
        tiling = {"encoder": eng.codec_tiling(False, T), "decoder": eng.codec_tiling(True, T)}
        wins = window_layout([T], Tw) if T > Tw else []
        groups = len(window_groups(len(wins), 1, Tw, window_rows_budget())) if wins else 0

        def run():
            out = model.separate(proc(descriptions=["dog barking"], audios=aud).to("cuda"), noise=noise)
            torch.cuda.synchronize()
            return out
        out = run()                                         # warm-up: plans, graph capture
        finite = bool(torch.isfinite(out.target[0]).all() and torch.isfinite(out.residual[0]).all())
        del out
        xs = []
        for _ in range(args.rounds):
            t0 = time.perf_counter()
            run()
            xs.append(time.perf_counter() - t0)
        med, lo, hi = summary(xs)
        row = {"clip_s": seconds, "T": T, "windows": len(wins), "groups": groups, "separate_s_median": round(med, 3),
               "s_range": [round(lo, 3), round(hi, 3)], "rtf": round(med / seconds, 5), "finite": finite,
               "workspace_bytes": eng.workspace_bytes(), "torch_peak_bytes": torch.cuda.max_memory_allocated(),
               "codec_tiling_halo_tile_frames": tiling}
        res["separate"].append(row)
        print(f"{seconds:5d} s clip separate() end to end: median {med:.3f} s (range {lo:.3f} .. {hi:.3f}), "
              f"real-time factor {row['rtf']:.5f} (wall / audio), {len(wins)} windows in {groups} groups, "
              f"finite={finite}, engine workspace {row['workspace_bytes'] / 1e9:.2f} GB, codec (halo, tile) {tiling}",
              flush=True)


def bench_window_plan(args, res, model, cfg):
    """DiT workspace of one group at the default row budget: a fresh engine (weights only) prepared for a group of
    budget / Tw windows; the difference is the group's plan."""
    from sam_audio_b200.windows import DEFAULT_WINDOW_ROWS
    Tw = cfg.transformer.max_positions
    n = max(1, DEFAULT_WINDOW_ROWS // Tw)
    eng = model._ensure_engine()
    w0 = eng.workspace_bytes()
    feats = torch.zeros(n, Tw, 256, device="cuda")
    text = torch.zeros(n, 4, 768, device="cuda")
    ids = torch.tensor([[0, 3]] * n, device="cuda")
    al = torch.zeros(n, Tw, dtype=torch.long, device="cuda")
    model._install_conditioning(feats, text, None, None, ids, al, None)
    torch.cuda.synchronize()
    plan = eng.workspace_bytes() - w0
    res["window_group_plan"] = {"windows": n, "rows": n * Tw, "dit_plan_bytes": plan,
                                "bytes_per_row": round(plan / (n * Tw))}
    print(f"DiT plan of one window group at the default budget ({n} windows x {Tw} frames = {n * Tw} rows): "
          f"{plan / 1e9:.2f} GB ({plan / (n * Tw) / 1e3:.1f} KB per row)", flush=True)


def bench_blend(args, res):
    """sab_blend_windows alone, CUDA events over many launches, at the shape of a 30 min clip (5 windows of 10 000
    frames into 45 000): HBM bytes = every window row read once + every output frame written once."""
    from sam_audio_b200 import _capi
    from sam_audio_b200.windows import window_layout, window_ramp
    Tw, T = 10000, 45000
    wins = window_layout([T], Tw)
    win = torch.randn(len(wins), Tw, 256, device="cuda")
    seq = torch.zeros(len(wins), dtype=torch.int32, device="cuda")
    start = torch.tensor([w.start for w in wins], dtype=torch.int32, device="cuda")
    flags = torch.tensor([_capi.WIN_FIRST * w.first + _capi.WIN_LAST * w.last for w in wins], dtype=torch.uint8,
                         device="cuda")
    out = torch.empty(1, T, 256, device="cuda")
    nbytes = (win.numel() + out.numel()) * 4.0
    xs = [timed(lambda: _capi.blend_windows(win, seq, start, flags, window_ramp(Tw), out), args.warmup, args.iters,
                args.min_window) for _ in range(args.rounds)]
    med, lo, hi = summary(xs)
    row = {"windows": len(wins), "Tw": Tw, "T": T, "ms_median": round(med, 4), "ms_range": [round(lo, 4), round(hi, 4)],
           "GBps": round(nbytes / (med * 1e-3) / 1e9, 1), "share_of_hbm": round(nbytes / (med * 1e-3) / PEAK_HBM, 3)}
    res["blend"] = row
    print(f"blend_windows {len(wins)} x {Tw} -> {T} frames: median {med:.4f} ms (range {lo:.4f} .. {hi:.4f}), "
          f"{row['GBps']:.1f} GB/s = {row['share_of_hbm']:.3f} of 3.35 TB/s", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--min-window", type=float, default=0.25, help="seconds of GPU work per timing window")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model", default="sam-audio-large")
    ap.add_argument("--skip-steps", action="store_true")
    ap.add_argument("--clips", default="300", help="comma-separated clip lengths (s) for the separate() arm")
    ap.add_argument("--only-separate", action="store_true",
                    help="only the window blend kernel, the window group's plan and the separate() arm")
    args = ap.parse_args()
    args.clips = [int(x) for x in args.clips.split(",")]
    assert torch.cuda.is_available(), "longform_bench needs a GPU"
    import __graft_entry__ as g
    g.build()
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    res = {"device": name, "power_limit": limit, "model": args.model, "kernels": [], "steps": []}
    if args.only_separate:
        from sam_audio_b200.config import stand_in_config
        from sam_audio_b200.model import SAMAudio
        from sam_audio_b200.synthetic import make_state_dict
        from sam_audio_b200.text_encoder import SyntheticTextEncoder
        bench_blend(args, res)
        cfg = stand_in_config(args.model)
        m = SAMAudio(cfg, text_encoder=SyntheticTextEncoder())
        m.load_state_dict(make_state_dict(cfg, seed=0, device="cuda"))
        m = m.eval().cuda()
        m._ensure_engine()
        m._state = None
        torch.cuda.empty_cache()
        bench_window_plan(args, res, m, cfg)
        bench_separate(args, res, m, cfg)
    else:
        bench_kernels(args, res)
        if not args.skip_steps:
            bench_steps(args, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
