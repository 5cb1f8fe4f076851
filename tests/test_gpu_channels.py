"""GPU (H100) tests of the multichannel stems (sab_spread_channels, sam_audio_b200/csrc/spread_channels.cuh;
SAMAudio.spread_channels(); keep_channels streams, groups and jobs in sam_audio_b200/stream.py).

The kernel is checked against a float64 restatement of its definition with torch.fft (rel-L2 <= 1e-5 per channel: fp32
radix-2 FFTs of 2048 points lose about log2(N) u relative to the spectrum's norm, ~1e-6).  The random-weight stand-ins
make no meaningful separation, so the stream tests check the construction: chunking invariance, the composition with
the mono stream, and that the mono path keeps its bits."""
import math
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

DESC = "a piano"
A, N = 512, 2048
U = 2.0 ** -24


@pytest.fixture(scope="module")
def eng(tiny_model):
    return tiny_model._ensure_engine()


@pytest.fixture(scope="module")
def small_model(tiny_model):
    from sam_audio_b200.model import build_synthetic_model
    return build_synthetic_model("sam-audio-small", seed=0, device="cuda:0", weights_device="cuda:0")


def _reference(t, r, x, Sp):
    """float64 (target [C, S'], residual [C, S']) of the definition, for t, r [S'] and x [C, S] (zero past S)."""
    t, r, x = t.double().cpu(), r.double().cpu(), x.double().cpu()
    C, S = x.shape
    n_frames = (Sp - 1) // A + 4
    L = 3 * A + n_frames * A + A                       # samples [-3a, n_frames a + a)
    def frames(sig):                                   # [rows, n_frames, N]
        buf = torch.zeros(sig.shape[0], L, dtype=torch.float64)
        buf[:, 3 * A:3 * A + sig.shape[1]] = sig
        return buf.unfold(1, N, A)[:, :n_frames]
    n = torch.arange(N, dtype=torch.float64)
    w = 0.5 - 0.5 * torch.cos(2 * math.pi * n / N)
    T = torch.fft.rfft(frames(t[None]) * w, dim=-1)[0]
    R = torch.fft.rfft(frames(r[None]) * w, dim=-1)[0]
    M = (T.abs() ** 2 + 1e-10) / (T.abs() ** 2 + R.abs() ** 2 + 2e-10)
    y = torch.fft.irfft(M * torch.fft.rfft(frames(x) * w, dim=-1), n=N, dim=-1) * w     # [C, n_frames, N]
    acc = torch.zeros(C, L, dtype=torch.float64)
    for j in range(n_frames):
        acc[:, j * A:j * A + N] += y[:, j]
    tgt = acc[:, 3 * A:3 * A + Sp] * (2.0 / 3.0)
    xp = torch.zeros(C, Sp, dtype=torch.float64)
    xp[:, :S] = x
    return tgt, xp - tgt


def _signal(rows, L, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(rows, L, generator=g) * torch.exp(torch.randn(rows, 1, generator=g))


def _rel(a, b):
    return float((a.double().cpu() - b).norm() / b.norm().clamp_min(1e-300))


@pytest.mark.parametrize("C", [1, 2, 6, 8])
@pytest.mark.parametrize("Sp,S", [(48_000, 48_000), (30_011, 29_000), (1500, 1500), (700, 300), (2048 * 5 + 77, 9000)])
def test_kernel_against_float64(tiny_model, C, Sp, S):
    """SAMAudio.spread_channels against the float64 definition: lengths that are not multiples of a, shorter than N, and
    S < S'.  Rel-L2 <= 1e-5 per channel for target and residual, and the residual is the mixture minus the target in
    one fp32 rounding."""
    tr = _signal(2, Sp, Sp + C)
    t, r = tr[0].cuda(), (0.5 * tr[1]).cuda()
    x = _signal(C, S, 7 * C + S).cuda()
    tgt, res = tiny_model.spread_channels(t, r, x)
    torch.cuda.synchronize()
    assert tgt.shape == res.shape == (C, Sp)
    ref_t, ref_r = _reference(t, r, x, Sp)
    for c in range(C):
        assert _rel(tgt[c], ref_t[c]) <= 1e-5, (c, _rel(tgt[c], ref_t[c]))
        assert _rel(res[c], ref_r[c]) <= 1e-5, (c, _rel(res[c], ref_r[c]))
    xp = torch.zeros(C, Sp, dtype=torch.float64)
    xp[:, :S] = x.double().cpu()
    td, rd = tgt.double().cpu(), res.double().cpu()
    assert torch.all((td + rd - xp).abs() <= U * (xp - td).abs())


@pytest.mark.parametrize("C", [1, 2, 6])
def test_zero_residual_reproduces_the_mixture(tiny_model, C):
    """With R = 0 the mask is 1 up to 1e-10 / |T|^2 and the target is the mixture within FFT rounding; the stems sum to
    the mixture within one fp32 rounding everywhere."""
    S = 40_000 + 123
    t = _signal(1, S, 3)[0].cuda()
    x = _signal(C, S, 4 + C).cuda()
    tgt, res = tiny_model.spread_channels(t, torch.zeros_like(t), x)
    torch.cuda.synchronize()
    xd, td, rd = x.double().cpu(), tgt.double().cpu(), res.double().cpu()
    for c in range(C):
        assert _rel(tgt[c], xd[c]) <= 1e-5
    assert torch.all((td + rd - xd).abs() <= U * (xd - td).abs())


def _seg(t, r, x, tr_first, tr_length, x_first, x_length, ot, orr, q0, q1):
    return dict(channels=x.shape[0], target=t.data_ptr(), residual=r.data_ptr(), tr_first=tr_first,
                tr_count=t.shape[0], tr_length=tr_length, mix=x.data_ptr(), mix_channel_stride=x.stride(0),
                mix_first=x_first, mix_count=x.shape[1], mix_length=x_length, out_target=ot.data_ptr(),
                out_residual=orr.data_ptr(), out_channel_stride=ot.stride(0), out_first=q0, out_count=q1 - q0)


@pytest.mark.parametrize("C", [2, 6])
def test_any_segmentation_gives_the_same_bits(eng, C):
    """One call cut into random output ranges, each reading buffers that hold only its input span (some with the lengths
    not known yet), in one launch and in one launch per range, is bit-equal to one segment over the whole signal."""
    from sam_audio_b200.channels import input_span
    rng = random.Random(C)
    Sp, S = 60_000 + 321, 59_000
    tr = _signal(2, Sp, 11).cuda()
    t, r = tr[0].contiguous(), tr[1].contiguous()
    x = _signal(C, S, 12).cuda()
    whole = torch.empty(2, C, Sp, device="cuda")
    eng.spread_channels([_seg(t, r, x, 0, Sp, 0, S, whole[0], whole[1], 0, Sp)])
    for one_launch in (True, False):
        cuts = sorted(set([0, Sp] + [rng.randrange(1, Sp) for _ in range(rng.randrange(5, 30))]))
        got = torch.full((2, C, Sp), float("nan"), device="cuda")
        segs, keep = [], []
        for q0, q1 in zip(cuts, cuts[1:]):
            i0, i1 = input_span(q0, q1)
            i0 = max(0, i0)
            unknown = i1 <= S and rng.random() < 0.5          # as a stream before its flush: the window holds all
            ts, rs = t[i0:min(i1, Sp)].contiguous(), r[i0:min(i1, Sp)].contiguous()
            xs = x[:, min(i0, S):min(i1, S)].contiguous()
            keep += [ts, rs, xs]
            segs.append(_seg(ts, rs, xs, i0, -1 if unknown else Sp, min(i0, S), -1 if unknown else S, got[0, :, q0:q1],
                             got[1, :, q0:q1], q0, q1))
        if one_launch:
            eng.spread_channels(segs)
        else:
            for s in segs:
                eng.spread_channels([s])
        torch.cuda.synchronize()
        assert torch.equal(got, whole)


# ---- streams ----
def _audio(C, seconds, rate, seed):
    from sam_audio_b200.synthetic import synthetic_clip
    return torch.stack([synthetic_clip(seed + c, int(rate * seconds), sr=rate)[0] for c in range(C)]).cuda()


def _sizes(n, seed):
    rng = random.Random(seed)
    sizes, total = [], 0
    while total < n:
        s = rng.choice([1, 7, 159, 441, 1921, 4801, 16_001, 44_100, 100_003])
        sizes.append(s)
        total += s
    return sizes


def _run(model, x, sizes, rate, keep, ws=2.0, seed=0):
    s = model.stream(DESC, window_seconds=ws, seed=seed, sample_rate=rate, keep_channels=keep)
    outs, i = [], 0
    for n in sizes:
        if i >= x.shape[-1]:
            break
        outs.append(s.push(x[..., i:i + n]))
        i += n
    outs.append(s.flush())
    torch.cuda.synchronize()
    return torch.cat([o.target for o in outs], -1), torch.cat([o.residual for o in outs], -1)


def _mean(x):
    """The channel mean as the resampler stages it: ascending sum, then one true division (a tensor divisor: PyTorch
    multiplies by the reciprocal of a Python scalar, which rounds differently for C = 6)."""
    m = x[0].clone()
    for c in range(1, x.shape[0]):
        m = m + x[c]
    return m / torch.full_like(m, x.shape[0]) if x.shape[0] > 1 else m


def _composition(model, x, rate, ws=2.0, seed=0):
    """resample(spread(T48, R48, x48_c), 48000, rate), T48 / R48 from the 48 kHz mono stream pushed whole."""
    x48m = x[0] if x.shape[0] == 1 and rate == 48000 else model.resample(_mean(x), rate, 48000)
    t48, r48 = _run(model, x48m, [x48m.numel()], 48000, False, ws, seed)
    x48 = model.resample(x, rate, 48000)
    tgt, res = model.spread_channels(t48, r48, x48)
    return model.resample(tgt, 48000, rate), model.resample(res, 48000, rate)


@pytest.mark.parametrize("which,rate,C", [("tiny", 48000, 2), ("tiny", 16000, 2), ("tiny", 44100, 6),
                                          ("small", 16000, 2)])
def test_keep_channels_stream_equals_the_composition(request, which, rate, C):
    """Three chunkings give identical [C, S] bits, equal to the composition of the mono stream, spread_channels and the
    resamplers; the same stream without keep_channels returns the mono stream's bits."""
    model = request.getfixturevalue("tiny_model" if which == "tiny" else "small_model")
    x = _audio(C, 7.3, rate, 5)
    runs = [_run(model, x, _sizes(x.shape[1], k), rate, True) for k in range(3)]
    for t, r in runs[1:]:
        assert torch.equal(t, runs[0][0]) and torch.equal(r, runs[0][1])
    t, r = _composition(model, x, rate)
    assert runs[0][0].shape == t.shape and t.shape[0] == C
    assert torch.equal(runs[0][0], t) and torch.equal(runs[0][1], r)
    mono = _run(model, x, _sizes(x.shape[1], 9), rate, False)
    x48m = x[0] if C == 1 and rate == 48000 else model.resample(_mean(x), rate, 48000)
    t48, r48 = _run(model, x48m, [x48m.numel()], 48000, False)
    assert torch.equal(mono[0], model.resample(t48, 48000, rate)) and torch.equal(mono[1], model.resample(r48, 48000,
                                                                                                            rate))


def test_a_group_mixing_keep_channels_and_mono(tiny_model):
    """Two keep-channels streams (48 kHz stereo, 16 kHz six channels) and two mono streams, 0.5 s per tick: every
    stream is bit-identical to itself alone; steady ticks build no plan and capture no graph, the workspace stays
    constant, and each tick makes one sab_spread_channels call."""
    from sam_audio_b200 import _capi
    specs = [(48000, 2, True), (16000, 6, True), (48000, 1, False), (16000, 2, False)]
    wavs = [_audio(C, 12.0, r, 20 + i) for i, (r, C, _) in enumerate(specs)]
    eng = tiny_model._ensure_engine()
    lib = _capi.lib()
    real = lib.sab_spread_channels
    calls = []
    g = tiny_model.stream_group(window_seconds=2.0)
    streams = [g.open(DESC, seed=i, sample_rate=r, keep_channels=k) for i, (r, _, k) in enumerate(specs)]
    outs, chunks = [[] for _ in specs], [[] for _ in specs]
    stats = []
    n_ticks = 24
    cur = [0]
    for tick in range(n_ticks):
        cur[0] = tick
        push = {}
        for i, ((rate, _, _), w) in enumerate(zip(specs, wavs)):
            c = w[:, tick * rate // 2:(tick + 1) * rate // 2]
            chunks[i].append(c)
            push[streams[i]] = c
        if tick == n_ticks // 2:
            torch.cuda.synchronize()
            stats.append((eng.plan_stats(), eng.workspace_bytes()))
            lib.sab_spread_channels = lambda *a: calls.append(cur[0]) or real(*a)
        res = g.push(push)
        for i, s in enumerate(streams):
            outs[i].append(res[s])
    torch.cuda.synchronize()
    stats.append((eng.plan_stats(), eng.workspace_bytes()))
    lib.sab_spread_channels = real
    tails = g.close()
    p0, p1 = stats[0][0], stats[1][0]
    assert p1["dit_plan_builds"] == p0["dit_plan_builds"] and p1["graph_captures"] == p0["graph_captures"]
    assert p1["codec_plan_builds"] == p0["codec_plan_builds"] and stats[1][1] == stats[0][1]
    assert calls and len(calls) == len(set(calls))             # at most one call per tick
    for i, (rate, C, keep) in enumerate(specs):
        outs[i].append(tails[streams[i]])
        t, r = torch.cat([o.target for o in outs[i]], -1), torch.cat([o.residual for o in outs[i]], -1)
        s = tiny_model.stream(DESC, window_seconds=2.0, seed=i, sample_rate=rate, keep_channels=keep)
        alone = [s.push(c) for c in chunks[i]] + [s.flush()]
        assert torch.equal(t, torch.cat([o.target for o in alone], -1)), i
        assert torch.equal(r, torch.cat([o.residual for o in alone], -1)), i
        assert t.dim() == (2 if keep else 1)


@pytest.mark.parametrize("rate,C", [(16000, 2), (48000, 2)])
def test_keep_channels_job_equals_the_stream_pushed_whole(tiny_model, rate, C):
    wav = _audio(C, 20.0, rate, 3)
    g = tiny_model.stream_group(window_seconds=2.0)
    job = g.submit(wav, DESC, seed=5, sample_rate=rate, keep_channels=True)
    g.drain()
    g.close()
    out = job.result()
    t, r = _run(tiny_model, wav, [wav.shape[1]], rate, True, seed=5)
    assert out.target.shape == t.shape and t.shape[0] == C
    assert torch.equal(out.target, t) and torch.equal(out.residual, r)


def test_memory_is_bounded_with_keep_channels(tiny_model):
    """1 s pushes of 16 kHz stereo with keep_channels at W = 50: the engine's workspace and the allocator's peak after
    20 windows equal those after 3."""
    x = _audio(2, 40.0, 16000, 40)
    s = tiny_model.stream(DESC, window_seconds=2.0, sample_rate=16000, keep_channels=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    at = {}
    for i in range(0, x.shape[1], 16000):
        s.push(x[:, i:i + 16000])
        if s.windows_solved in (3, 20) and s.windows_solved not in at:
            torch.cuda.synchronize()
            at[s.windows_solved] = (s.workspace_bytes(), torch.cuda.max_memory_allocated())
    s.flush()
    assert set(at) == {3, 20}
    assert at[20] == at[3]
