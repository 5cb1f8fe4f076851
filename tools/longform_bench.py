"""Long-form (T > 256 latent frames) self-attention on the sam-audio-large stand-in, two measurements in one run:

  1. kernels alone, through the C-ABI seams, CUDA events over many launches: the wgmma streaming kernel
     (attention_stream_tc.cuh; bounded and exact softmax) against the mma.sync streaming kernel (attention.cuh) on the
     same shapes, T in {750, 3000, 7500} (30 s, 2 min, 5 min), 22 heads, items chosen so the grid fills the card
     several times over;
  2. one midpoint ODE step (two DiT evaluations, every kernel of the layer stack) of one clip of 30 s and of 5 min,
     default engine against an engine planned under SAB_NO_TC_ATTENTION=1, alternated, every shape warmed up;
  3. separate() of one 5 min clip end to end on the default engine (codec encode in time tiles, 32 evaluations, codec
     decode in time tiles), with the engine's workspace_bytes afterwards and the tile lengths the codec chose.

Every timing window is stretched to at least --min-window seconds of GPU work; a row quotes the median of the rounds and
their range.  The kernel rows go through the test seams, which encode three TMA descriptors on the host per call: for
the shortest kernel (T = 750) the host may not keep the GPU busy, and the row is then a lower bound on the kernel's rate.

Achieved TFLOP/s counts 4 * T^2 * 128 per (item, head).  The floor is the larger of FLOPs / 989 TFLOP/s (H100 SXM data
sheet, dense bf16, 700 W) and q|k|v|o once / 3.35 TB/s; the line says which of the two it is.  Prints the card name and
its power limit, and one JSON line at the end.  Fails without a GPU.

    python tools/longform_bench.py [--min-window 0.25] [--model sam-audio-large]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys

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
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_noise
    hop, sr = cfg.audio_codec.hop_length, cfg.audio_codec.sample_rate
    seconds = 300
    T = seconds * sr // hop
    proc = SAMAudioProcessor(hop, sr)
    aud = [synthetic_clip(11, seconds * sr)]
    noise = synthetic_noise(1, T).cuda()
    eng = model._ensure_engine()
    tiling = {"encoder": eng.codec_tiling(False, T), "decoder": eng.codec_tiling(True, T)}

    def run():
        return model.separate(proc(descriptions=["dog barking"], audios=aud).to("cuda"), noise=noise)
    out = run()                                             # warm-up: plans, graph capture
    torch.cuda.synchronize()
    finite = bool(torch.isfinite(out.target[0]).all() and torch.isfinite(out.residual[0]).all())
    xs = []
    for _ in range(args.rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run()
        e1.record()
        torch.cuda.synchronize()
        xs.append(e0.elapsed_time(e1) * 1e-3)
    med, lo, hi = summary(xs)
    row = {"clip_s": seconds, "T": T, "separate_s_median": round(med, 3), "s_range": [round(lo, 3), round(hi, 3)],
           "samples": int(out.target[0].numel()), "finite": finite, "workspace_bytes": eng.workspace_bytes(),
           "torch_peak_bytes": torch.cuda.max_memory_allocated(),
           "codec_tiling_halo_tile_frames": tiling}
    res["separate"] = row
    print(f"{seconds:4d} s clip separate() end to end: median {med:.3f} s (range {lo:.3f} .. {hi:.3f}), finite={finite}, "
          f"engine workspace {row['workspace_bytes'] / 1e9:.2f} GB, codec (halo, tile) frames {tiling}", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--min-window", type=float, default=0.25, help="seconds of GPU work per timing window")
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--model", default="sam-audio-large")
    ap.add_argument("--skip-steps", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "longform_bench needs a GPU"
    import __graft_entry__ as g
    g.build()
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    res = {"device": name, "power_limit": limit, "model": args.model, "kernels": [], "steps": []}
    bench_kernels(args, res)
    if not args.skip_steps:
        bench_steps(args, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
