"""bench.py — separated clips/sec of SAMAudio.separate() (10 s @ 48 kHz clips) on N H100s.

    python bench.py --gpus 1 --steps 3 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N --steps K --warmup W
    python bench.py --impl reference ...      # the reference algorithm's CPU path (oracle port) on host cores

One "step" = one separate() over a batch of B synthetic clips per GPU (weak scaling): DAC-VAE encode,
conditioning, 32 DiT evaluations (midpoint ODE), DAC-VAE decode of target+residual, and — for N>1 — the
all-gather of the separated waveforms.  Prints ONE JSON line (rank 0).

    python bench.py ... --dump-outputs DIR    # after the timed steps: DIR/target.npy, DIR/residual.npy (float32)

With the same arguments the inputs (weights, clips, noise) are identical from run to run, so two builds can be
compared output for output.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "separated clips/sec (10s@48kHz, sam-audio-large) at 1/2/4/8 H100 vs ref CPU"
UNIT = "clips/s"


def _peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        d = json.load(open(p))
        return dict(hbm=float(d["hbm_gbs"]), tf_burst=float(d["bf16_tflops"]),
                    tf_sustained=float(d.get("bf16_tflops_sustained", d["bf16_tflops"])), source="measured")
    # NVIDIA H100 SXM data sheet (700 W): 3.35 TB/s HBM3, 989 dense BF16 TFLOP/s — a bound, not a measured rate
    return dict(hbm=3350.0, tf_burst=989.0, tf_sustained=989.0, source="H100 SXM data sheet")


class ClockSampler:
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.f = tempfile.NamedTemporaryFile("w+", suffix=".csv", delete=False)
        self.idx = gpu_index
        try:
            self.p = subprocess.Popen(["nvidia-smi", f"--id={gpu_index}", f"--query-gpu={self.Q}",
                                       "--format=csv,noheader,nounits", "-lms", "200"], stdout=self.f,
                                      stderr=subprocess.DEVNULL)
        except Exception:
            self.p = None

    def stop(self):
        if self.p is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.p.terminate()
        try:
            self.p.wait(5)
        except Exception:
            self.p.kill()
        self.f.flush()
        rows = [r.strip().split(", ") for r in open(self.f.name) if r.strip()]
        os.unlink(self.f.name)
        sm, mx, pw, reasons = [], 0.0, [], set()
        for r in rows:
            try:
                sm.append(float(r[1]))
                mx = max(mx, float(r[2]))
                pw.append(float(r[3]))
                for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[5:9]):
                    if v.strip().lower() == "active":
                        reasons.add(name)
            except Exception:
                continue
        # "under load" = samples drawing clearly more than idle power
        hot = [s for s, p in zip(sm, pw) if p > 300] or sm
        return {"sm_mhz": statistics.median(hot) if hot else None, "sm_max_mhz": mx or None,
                "power_w_max": max(pw) if pw else None, "samples": len(rows), "reasons": sorted(reasons)}


def _dist_setup(n_gpus: int):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    assert world == n_gpus or world == 1, f"--gpus {n_gpus} but WORLD_SIZE={world}"
    return world, rank, local


# ------------------------------------------------------------------------------------------------
# CPU legs (oracle port): bounded sample of the same workload
# ------------------------------------------------------------------------------------------------
def pick_cpu_threads():
    """All the host threads the process can actually use: the smaller of the affinity mask and the cgroup CPU
    quota, then a 1-2 s fp32 GEMM probe over {that, half, quarter, ...} picks the fastest setting (a container
    that reports 128 logical CPUs but is throttled by a quota runs fastest with fewer threads)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    for quota_file, period_file in (("/sys/fs/cgroup/cpu.max", None),
                                    ("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "/sys/fs/cgroup/cpu/cpu.cfs_period_us")):
        try:
            if period_file is None:
                q, per = open(quota_file).read().split()
            else:
                q, per = open(quota_file).read().strip(), open(period_file).read().strip()
            if q not in ("max", "-1"):
                n = max(1, min(n, int(float(q) / float(per) + 0.5)))
            break
        except Exception:
            continue
    a = torch.randn(250, 2816)
    b = torch.randn(2816, 7552)
    best, best_t = n, None
    cand = sorted({max(1, n >> s) for s in range(0, 5)}, reverse=True)
    for c in cand:
        torch.set_num_threads(c)
        for _ in range(3):
            torch.mm(a, b)                                  # thread-pool spin-up / first touch
        dt = 1e9
        for _ in range(3):
            t0 = time.perf_counter()
            for _ in range(3):
                torch.mm(a, b)
            dt = min(dt, time.perf_counter() - t0)
        if best_t is None or dt < 0.95 * best_t:             # prefer more threads unless clearly slower
            best, best_t = c, dt
    torch.set_num_threads(best)
    return best, n


def cpu_full_clip(sd, cfg, n_threads: int):
    """ONE clip through the whole path on the host cores (no extrapolation): encode, all 16 midpoint steps
    (32 evaluations), decode.  Returns seconds."""
    from oracle import restate
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_noise, synthetic_text_features
    torch.set_num_threads(n_threads)
    torch.set_grad_enabled(False)
    cc = cfg.audio_codec
    wav = synthetic_clip(0)[None]
    tf, tm = synthetic_text_features(["man speaking"])
    T = wav.shape[-1] // cc.hop_length
    mask = torch.ones(1, T, dtype=torch.bool)
    ids, al = restate.process_anchors(None, mask, cc.hop_length, cc.sample_rate)
    t0 = time.perf_counter()
    restate.separate(sd, cfg, wav, mask, torch.tensor([float(T)]), tf, tm, ids, al, synthetic_noise(1, T))
    return time.perf_counter() - t0


def cpu_sample(sd, cfg, n_threads: int, repeats: int = 1):
    """One clip of the workload on the host cores through the oracle port (fp32 torch, the reference's
    algorithm): encode once + ONE of the 16 midpoint steps (2 DiT evaluations) + decode target & residual.
    clips/s = 1 / (t_encode + 16 * t_step + t_decode).  Returns (clips_per_s, detail)."""
    from oracle import restate
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_noise, synthetic_text_features
    torch.set_num_threads(n_threads)
    torch.set_grad_enabled(False)
    cc = cfg.audio_codec
    wav = synthetic_clip(0)[None]                                   # [1,1,480000]
    tf, tm = synthetic_text_features(["man speaking"])
    best = None
    for _ in range(repeats):
        t0 = time.perf_counter()
        feats = restate.codec_encode(sd, cc, wav).transpose(1, 2)
        feats = torch.cat([feats, feats], 2)
        t1 = time.perf_counter()
        T = feats.shape[1]
        mask = torch.ones(1, T, dtype=torch.bool)
        ids, al = restate.process_anchors(None, mask, cc.hop_length, cc.sample_rate)
        video = feats.new_zeros(1, cfg.vision_encoder.dim, T)
        y = synthetic_noise(1, T)

        def field(t, yy):
            return restate.samaudio_forward(sd, cfg, yy, feats, tf, t.expand(1), video, tm, ids, al, mask)
        dt = 1.0 / 16
        f0 = field(torch.tensor(0.0), y)
        f1 = field(torch.tensor(dt / 2), y + f0 * (dt / 2))
        y = y + dt * f1
        t2 = time.perf_counter()
        w = restate.codec_decode(sd, cc, y.transpose(1, 2).reshape(2, cc.codebook_dim, T))
        t3 = time.perf_counter()
        assert w.shape[-1] == 480000
        d = dict(encode_s=t1 - t0, ode_step_s=t2 - t1, decode_s=t3 - t2)
        d["clip_s"] = d["encode_s"] + 16 * d["ode_step_s"] + d["decode_s"]
        if best is None or d["clip_s"] < best["clip_s"]:
            best = d
        _CPU_SAMPLE_OUT.update(features=feats[:, :, : cc.codebook_dim], velocity=f1, latent=y, wav=w.view(2, -1))
    return 1.0 / best["clip_s"], best


_CPU_SAMPLE_OUT = {}          # tensors of the last cpu_sample(): what the GPU parity gate is checked against


def gpu_sample(model, cfg, dev):
    """The SAME bounded sample as cpu_sample() (clip 0, prompt, noise; encode + one midpoint step of 1/16 + decode)
    through the CUDA path — the parity gate of the bench line compares the two."""
    from oracle import restate
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_noise, synthetic_text_features
    cc = cfg.audio_codec
    with torch.inference_mode():
        feats = model._get_audio_features(synthetic_clip(0)[None].to(dev))
        tf, tm = synthetic_text_features(["man speaking"])
        T = feats.shape[1]
        mask = torch.ones(1, T, dtype=torch.bool)
        ids, al = restate.process_anchors(None, mask, cc.hop_length, cc.sample_rate)      # integer host logic
        model._install_conditioning(feats, tf.to(dev), tm.to(dev), None, ids.to(dev), al.to(dev), mask.to(dev))
        eng = model._ensure_engine()
        y = synthetic_noise(1, T).to(dev)
        dt = 1.0 / 16
        f0, f1 = torch.empty_like(y), torch.empty_like(y)
        eng.dit_forward(y, torch.zeros(1, device=dev), f0)
        eng.dit_forward((y + f0 * (dt / 2)).contiguous(), torch.full((1,), dt / 2, device=dev), f1)
        y1 = (y + dt * f1).contiguous()
        w = torch.empty(1, 2, T * cc.hop_length, device=dev)
        eng.decode(y1, 1, T, w)
        torch.cuda.synchronize()
    return dict(features=feats[:, :, : cc.codebook_dim].cpu(), velocity=f1.cpu(), latent=y1.cpu(), wav=w[0].cpu())


PARITY_TOL = {"features_rel_l2": 2e-2, "velocity_rel_l2": 2e-2, "wav_snr_db": 30.0}


def parity_gate(gpu, cpu):
    import math

    def rl2(a, b):
        return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))
    r = {"features_rel_l2": rl2(gpu["features"], cpu["features"]),
         "velocity_rel_l2": rl2(gpu["velocity"], cpu["velocity"]),
         "latent_rel_l2": rl2(gpu["latent"], cpu["latent"]),
         "wav_snr_db": -20.0 * math.log10(max(rl2(gpu["wav"], cpu["wav"]), 1e-30))}
    r["rel_l2"], r["snr_db"] = r["velocity_rel_l2"], r["wav_snr_db"]
    r["tolerance"] = PARITY_TOL
    r["ok"] = bool(r["features_rel_l2"] <= PARITY_TOL["features_rel_l2"] and
                   r["velocity_rel_l2"] <= PARITY_TOL["velocity_rel_l2"] and r["wav_snr_db"] >= PARITY_TOL["wav_snr_db"])
    r["sample"] = ("clip 0 of the workload, same prompt and noise on both sides: DAC-VAE encode, one midpoint step of "
                   "1/16 (2 DiT evaluations at the benchmarked model shape), DAC-VAE decode; CUDA path vs the fp32 "
                   "CPU oracle (the cpu_baseline sample)")
    return r


SAMPLE_DESC = ("1 clip (10 s @ 48 kHz) through the oracle port on the host cores: DAC-VAE encode + 1 of the 16 "
               "midpoint steps (2 DiT evaluations, x16) + DAC-VAE decode of target+residual; fp32 torch")


def run_reference(args):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if world > 1 and rank != 0:
        return
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.synthetic import make_state_dict
    cores, avail = pick_cpu_threads()
    cfg = stand_in_config(args.model)
    sd = make_state_dict(cfg, seed=0)
    budget_s, t_start = 240.0, time.perf_counter()      # wall budget of this arm, the full clip included
    # one un-extrapolated clip (all 32 evaluations) first: it checks the x16 extrapolation of the bounded samples below
    full_s = cpu_full_clip(sd, cfg, cores) if args.steps >= 3 else None
    vals = []
    n_warm = 1 if args.warmup > 0 else 0                    # one untimed pass is enough to warm the CPU path
    n_total = n_warm + args.steps
    for i in range(n_total):
        v, d = cpu_sample(sd, cfg, cores)
        if i >= n_warm:
            vals.append((v, d))
        if i >= n_warm and time.perf_counter() - t_start > budget_s:
            break
    v = statistics.median([x[0] for x in vals])
    d = vals[0][1]
    line = {
        "impl": "reference", "metric": METRIC, "value": v, "unit": UNIT, "n_gpus": args.gpus, "steps": len(vals),
        "warmup": n_warm, "ms_per_step": 1e3 / v, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "f32", "data": "synthetic",
        # the GPU arm's workload at this N; the CPU leg times a bounded sample of it
        # (one clip of the batch, see cpu_baseline.sample): clips/s does not depend on which clip
        "config": _config(args, max(1, args.gpus), args.batch),
        "cpu_baseline": {"value": v, "unit": UNIT, "cores": cores, "cores_available": avail, "kind": "port",
                         "sample": SAMPLE_DESC, "detail_s": d,
                         "full_clip_s": full_s, "full_clip_note": "one clip through all 32 evaluations, not extrapolated "
                         "(null: skipped when --steps < 3); 1/full_clip_s should match `value`"},
        "e2e": {"value": v, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    print(json.dumps(line), flush=True)


def _config(args, world, batch):
    from sam_audio_b200.config import stand_in_config
    tc = stand_in_config(args.model).transformer
    return {
        "workload": f"{args.model} separate(): batch={batch}x10s@48kHz mono per GPU, text prompt, "
                    f"reranking_candidates={args.candidates} ({batch * args.candidates} ODE sequences per GPU; rankers "
                    f"None = candidate 0, config.py:214-215), predict_spans=False (PE-A-Frame span predictor is "
                    f"third-party and absent; "
                    f"at the pinned commit it does not change the audio), 16 midpoint steps = 32 DiT evaluations",
        "model_shape": f"stand-in (HF config.json is gated): dim={tc.dim} layers={tc.n_layers} heads={tc.n_heads} "
                       f"ffn={tc.ffn_hidden}; DAC-VAE 64/1024/1536 rates 2-8-10-12; random-init weights",
        "global_batch": world * batch, "candidates": args.candidates, "clip_seconds": 10, "sample_rate": 48000,
        "parallelism": f"dp{world}", "l2": "inputs_exceed_l2 (activations >> 50 MB)",
        "text_encoder": "t5-base shape, random init, hash tokenizer (no checkpoint on disk)",
    }


# ------------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------------
DUMP_CLIPS = 8     # 2 x 8 x 480000 fp32 = 31 MB


def dump_outputs(out_dir, out):
    """The waveforms separate() returned in the last timed step: a fixed, seeded sample of DUMP_CLIPS clips (all of
    them when there are fewer), target and residual, as [k, samples] float32 arrays in clip order."""
    import numpy as np
    if isinstance(out, torch.Tensor):                 # N > 1: the all-gathered [clips, 2, samples]
        target, residual = list(out[:, 0]), list(out[:, 1])
    else:
        target, residual = list(out.target), list(out.residual)
    n = len(target)
    pick = sorted(torch.randperm(n, generator=torch.Generator().manual_seed(0))[:DUMP_CLIPS].tolist())
    os.makedirs(out_dir, exist_ok=True)
    for name, wavs in (("target", target), ("residual", residual)):
        arr = torch.stack([wavs[i].detach().float().cpu() for i in pick]).numpy()
        np.save(os.path.join(out_dir, f"{name}.npy"), arr.astype(np.float32))
def run_gpu(args):
    import __graft_entry__ as g
    world, rank, local = _dist_setup(args.gpus)
    if rank == 0:
        import contextlib
        with contextlib.redirect_stdout(sys.stderr):      # stdout carries the ONE JSON line
            g.build()
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.parallel import all_gather_waveforms, broadcast_state_dict, separate_and_gather
    from sam_audio_b200.synthetic import (make_state_dict, synthetic_clip, synthetic_descriptions, synthetic_noise)
    from sam_audio_b200.text_encoder import T5TextEncoder

    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    cfg = stand_in_config(args.model)
    B, C = args.batch, args.candidates
    if args.global_batch:                      # strong scaling: a fixed global batch split over the ranks
        assert args.global_batch % world == 0, "--global-batch must be a multiple of the GPU count"
        B = args.global_batch // world
    # ---- weights: generated on rank 0, ONE broadcast over NCCL/NVLink ----
    sd = make_state_dict(cfg, seed=0, device=dev) if rank == 0 else None
    if world > 1:
        sd = broadcast_state_dict(sd, src=0, device=dev)
    model = SAMAudio(cfg, text_encoder=T5TextEncoder(cfg.text_encoder, allow_random_init=True))
    model.load_state_dict(sd)
    model = model.eval().to(dev)
    eng = model._ensure_engine()
    sd_cpu = None
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        sd_cpu = {k: v.float().cpu() for k, v in sd.items()}
    del sd
    model._state = None
    torch.cuda.empty_cache()
    # parity gate, GPU half (before the timed plan exists: a B=1 plan would otherwise evict the captured graph)
    gpu_par = gpu_sample(model, cfg, dev) if sd_cpu is not None else None

    proc = SAMAudioProcessor(cfg.audio_codec.hop_length, cfg.audio_codec.sample_rate)
    clips = [synthetic_clip(rank * B + i).pin_memory() for i in range(B)]
    desc = synthetic_descriptions(B)
    noise_host = synthetic_noise(B * C, 250, seed=4321 + rank).pin_memory()
    h2d = sum(c.numel() * 4 for c in clips) + noise_host.numel() * 4
    out_host = torch.empty(B, 2, 480000, dtype=torch.float32).pin_memory()
    d2h = out_host.numel() * 4

    def barrier():
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
        torch.cuda.synchronize()

    def gather_step(batch, noise):
        if args.gather == "overlap":   # the all-gather of each decoded chunk runs under the next chunk's decode
            return separate_and_gather(model, batch, noise, [B] * world, reranking_candidates=C)
        out = model.separate(batch, noise=noise, reranking_candidates=C)
        loc = torch.stack([torch.stack([t, r]) for t, r in zip(out.target, out.residual)])
        return all_gather_waveforms(loc, [B] * world)

    def step_resident(batch, noise):
        if world > 1:
            return gather_step(batch, noise)
        return model.separate(batch, noise=noise, reranking_candidates=C)

    def step_e2e():
        batch = proc(descriptions=desc, audios=clips)               # host: mono mix, pad, masks, anchors
        if not batch.audios.is_pinned():
            batch.audios = batch.audios.pin_memory()
        batch = batch.to(dev)                                       # H2D
        nz = noise_host.to(dev, non_blocking=True)
        if world > 1:
            full = gather_step(batch, nz)
            loc = full[rank * B:(rank + 1) * B]
        else:
            out = model.separate(batch, noise=nz, reranking_candidates=C)
            loc = torch.stack([torch.stack([t, r]) for t, r in zip(out.target, out.residual)])
        out_host.copy_(loc, non_blocking=True)                      # D2H of the step's result
        torch.cuda.current_stream().synchronize()
        return out_host

    batch_gpu = proc(descriptions=desc, audios=clips).to(dev)
    noise_gpu = noise_host.to(dev)
    for _ in range(max(args.warmup, 3)):
        step_resident(batch_gpu, noise_gpu)
    torch.cuda.synchronize()

    def timed(fn, k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        barrier()
        e0.record()
        for _ in range(k):
            if os.environ.get("BENCH_DEBUG"):
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                print(f"[rank {rank}] step {time.perf_counter() - t0:.3f} s", file=sys.stderr, flush=True)
            else:
                fn()
        e1.record()
        barrier()
        ms = torch.tensor([e0.elapsed_time(e1)], device=dev, dtype=torch.float64)
        if world > 1:
            import torch.distributed as dist
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms)

    sampler = ClockSampler(local) if rank == 0 else None
    # ---- value: inputs resident in HBM (the ODE solve replays as one CUDA graph) ----
    eng.launch_count(reset=True)
    last = {}
    ms_val = timed(lambda: last.__setitem__("out", step_resident(batch_gpu, noise_gpu)), args.steps)
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, last["out"])
    del last
    launches = eng.launch_count(reset=True)
    # ---- one more step with a CUDA event in front of every launch: live per-kernel times.  Every step replays the same
    #      captured graph, so one step gives the per-step breakdown; K more would only lengthen the run ----
    prof_steps = 1
    eng.profile(True)
    ms_prof = timed(lambda: step_resident(batch_gpu, noise_gpu), prof_steps)
    prof = eng.profile_report()
    eng.profile(False)
    eng.launch_count(reset=True)
    # ---- e2e: public API with HOST buffers (H2D of clips + noise, D2H of waveforms inside the region) ----
    step_e2e()
    ms_e2e = timed(step_e2e, args.steps)
    clocks = sampler.stop() if sampler else None

    if rank != 0:
        if world > 1:
            import torch.distributed as dist
            dist.destroy_process_group()
        return
    peaks = _peaks()
    clips_total = world * B * args.steps
    value = clips_total / (ms_val / 1e3)
    e2e = clips_total / (ms_e2e / 1e3)
    # dominant kernel = the wgmma GEMM (all DiT linears + codec convs): aggregate its launches
    # tensor-bound launches of the wgmma GEMM: algorithmic intensity above the ridge (peak FLOP/s / HBM bytes/s); the
    # weight-streaming launches below it (per-item bias GEMMs, text K/V, time embedders, 48 kHz codec stages) are
    # HBM-bound and reported under hbm_kernels instead
    ridge = peaks["tf_sustained"] * 1e12 / (peaks["hbm"] * 1e9)
    gemm_tags = [t for t in prof if not t.startswith(("sdpa", "rmsnorm", "codec.enc.conv0", "codec.dec.last"))
                 and prof[t]["flops"] > 0 and prof[t]["flops"] / max(prof[t]["bytes"], 1.0) >= ridge]
    g_ms = sum(prof[t]["ms"] for t in gemm_tags)
    g_fl = sum(prof[t]["flops"] for t in gemm_tags)
    g_n = sum(prof[t]["launches"] for t in gemm_tags)
    total_ms = sum(v["ms"] for v in prof.values())
    achieved = g_fl / (g_ms * 1e-3) / 1e12 if g_ms > 0 else 0.0
    groups = {"dit_gemm": 0.0, "codec_gemm": 0.0, "sdpa": 0.0, "norm_elementwise": 0.0, "codec_ends": 0.0}
    for t, v in prof.items():
        if t.startswith("sdpa"):
            groups["sdpa"] += v["ms"]
        elif t.startswith(("codec.enc.conv0", "codec.dec.last")):
            groups["codec_ends"] += v["ms"]
        elif t.startswith("codec."):
            groups["codec_gemm"] += v["ms"]
        elif v["flops"] > 0:
            groups["dit_gemm"] += v["ms"]
        else:
            groups["norm_elementwise"] += v["ms"]
    # HBM-bound kernels: algorithmic bytes per launch / live launch time vs the measured copy bandwidth
    hbm_tags = [t for t in prof if prof[t]["bytes"] > 0 and t not in gemm_tags]
    hbm = {t: {"launches_per_step": prof[t]["launches"] / prof_steps,
               "mb_per_launch": round(prof[t]["bytes"] / prof[t]["launches"] / 1e6, 2),
               "ms_per_step": round(prof[t]["ms"] / prof_steps, 3),
               "gbs": round(prof[t]["bytes"] / max(prof[t]["ms"], 1e-9) / 1e6, 1),
               "frac": round(prof[t]["bytes"] / max(prof[t]["ms"], 1e-9) / 1e6 / peaks["hbm"], 3)}
           for t in sorted(hbm_tags, key=lambda t: -prof[t]["ms"])}
    att = {t: v for t, v in prof.items() if t.startswith("sdpa")}
    att_tf = sum(v["flops"] for v in att.values()) / max(sum(v["ms"] for v in att.values()), 1e-9) / 1e9
    line = {
        "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": args.steps,
        "warmup": max(args.warmup, 3), "ms_per_step": ms_val / args.steps, "higher_is_better": True,
        "scaling": "strong" if args.global_batch else "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": _config(args, world, B),
        "e2e": {"value": e2e, "unit": UNIT, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                "ms_per_step": ms_e2e / args.steps},
        "gpu_launches": int(launches),
        "clocks": clocks,
        "roofline": {"kernel": "gemm_tc_kernel (wgmma segmented GEMM: launches above the roofline ridge = DiT linears "
                               "+ the wide codec convs)",
                     "bound": "tensor", "achieved": achieved, "peak": peaks["tf_sustained"], "unit": "TFLOP/s",
                     "frac": achieved / peaks["tf_sustained"],
                     "peak_source": peaks["source"],
                     "launches": int(g_n), "avg_launch_ms": g_ms / max(g_n, 1),
                     "share_of_step": g_ms / max(total_ms, 1e-9),
                     "profiled_ms_per_step": ms_prof / prof_steps,
                     "algorithmic_tflop_per_step": g_fl / 1e12 / prof_steps,
                     "dominant_launch": (lambda t: {"tag": t, "launches": int(prof[t]["launches"]),
                                                    "avg_launch_ms": prof[t]["ms"] / max(prof[t]["launches"], 1),
                                                    "tflop_per_launch": prof[t]["flops"] / max(prof[t]["launches"], 1) / 1e12,
                                                    "achieved": prof[t]["flops"] / max(prof[t]["ms"], 1e-9) / 1e9,
                                                    "frac": prof[t]["flops"] / max(prof[t]["ms"], 1e-9) / 1e9 / peaks["tf_sustained"]})(
                         max(gemm_tags, key=lambda t: prof[t]["ms"])) if gemm_tags else None},
        "breakdown_ms_per_step": {k: v / prof_steps for k, v in groups.items()},
        "hbm_kernels": {"peak_gbs": peaks["hbm"], "note": "algorithmic bytes (operands once + every epilogue stream "
                        "once) / live launch time, sustained inside the step", "kernels": hbm},
        "sdpa_tflops": att_tf,
        "kernels": {t: {"ms_per_step": round(v["ms"] / prof_steps, 3), "launches_per_step": v["launches"] / prof_steps,
                        "tflops": round(v["flops"] / max(v["ms"], 1e-9) / 1e9, 1)}
                    for t, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])},
        "workspace_gib": eng.workspace_bytes() / 2 ** 30,
    }
    if sd_cpu is not None:
        cores, avail = pick_cpu_threads()
        v, d = cpu_sample(sd_cpu, cfg, cores)
        line["cpu_baseline"] = {"value": v, "unit": UNIT, "cores": cores, "cores_available": avail, "kind": "port",
                                "sample": SAMPLE_DESC, "detail_s": d}
        # parity gate (BASELINE.md 3.5): no throughput is reported for a path whose results differ from the oracle's
        line["parity"] = parity_gate(gpu_par, _CPU_SAMPLE_OUT)
        if not line["parity"]["ok"]:
            for k in ("value", "ms_per_step"):
                line[k] = None
            line["e2e"]["value"] = None
            line["error"] = "parity gate failed: throughput withheld"
            print(json.dumps(line), flush=True)
            sys.exit(1)
    else:
        line["parity"] = {"checked": False, "why": "the CPU oracle leg runs on rank 0 at N=1 only (the same library and "
                                                   "kernels run at every N); see tests/test_gpu_parity_large.py"}
    print(json.dumps(line), flush=True)
    if world > 1:
        import torch.distributed as dist
        dist.destroy_process_group()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="cuda", choices=["cuda", "reference"])
    ap.add_argument("--model", default="sam-audio-large")
    ap.add_argument("--batch", type=int, default=64, help="clips per GPU per step")
    ap.add_argument("--candidates", type=int, default=1, help="reranking_candidates (BASELINE config 4: 8)")
    ap.add_argument("--global-batch", type=int, default=0,
                    help="strong scaling: total clips split over the GPUs (overrides --batch)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--gather", default="overlap", choices=["overlap", "after"],
                    help="N>1: all-gather each decoded chunk under the next chunk's decode, or once after the decode")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the separated waveforms of the last timed step (a fixed sample "
                         f"of at most {DUMP_CLIPS} clips) as DIR/target.npy and DIR/residual.npy, float32")
    a = ap.parse_args()
    if a.impl == "reference":
        run_reference(a)
    else:
        run_gpu(a)
