"""GPU (H100) tests of the resampler (sab_resample, sam_audio_b200/csrc/resample.cuh) and of streams at other rates and
channel counts (SAMAudio.stream(sample_rate=...), sam_audio_b200/stream.py).

Kernel bound.  Output y = sum_k w_k v_k with v_k the staged channel mean of input k and w_k the fp32 table entry (exact in
float64).  Staging sums C fp32 values in ascending order (C - 1 roundings, each at most u = 2^-24 of the partial sum, so
at most (C - 1) u sum_c |x_c|) and divides by C (one more rounding): |v - mean_c x_c| <= C u mean_c |x_c|, to first
order.  The chain of K FMAs rounds K times, each at most u of the partial sum, so |y - sum_k w_k v_k| <= K u
sum_k |w_k v_k|.  Together, to first order: |y - sum_k w_k mean_c x_ck| <= (K + C + 1) u sum_k |w_k| mean_c |x_ck|,
where the reference is the float64 sum over the same fp32 table and fp32 samples.
"""
import math
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

RATES = [8000, 11025, 16000, 22050, 32000, 44100, 96000, 192000]
PAIRS = [(r, 48000) for r in RATES] + [(48000, r) for r in RATES] + [(48000, 48000)]
DESC = "dog barking"
U = 2.0 ** -24
GUARD = 64


@pytest.fixture(scope="module")
def eng(tiny_model):
    return tiny_model._ensure_engine()


def _table(orig, new):
    from sam_audio_b200 import _capi
    K, lo, w = _capi.resample_taps(orig, new)
    g = math.gcd(orig, new)
    return orig // g, new // g, K, lo.astype(np.int64), w.astype(np.float64)


def _reference(x, orig, new, q0, q1, length):
    """float64 y[q0:q1] and its bound, for x [C, L] fp32 (cpu) with samples outside [0, length) zero."""
    o, n, K, lo, w = _table(orig, new)
    xd = x.double().numpy()
    mean, amean = xd.mean(0), np.abs(xd).mean(0)
    q = np.arange(q0, q1)
    j = q % n
    idx = ((q // n) * o + lo[j])[:, None] + np.arange(K)[None, :]
    valid = (idx >= 0) & (idx < length)
    v = np.where(valid, mean[np.clip(idx, 0, length - 1)], 0.0)
    a = np.where(valid, amean[np.clip(idx, 0, length - 1)], 0.0)
    C = x.shape[0]
    return (w[j] * v).sum(1), (K + C + 1) * U * (np.abs(w[j]) * a).sum(1) + 1e-30


def _signal(C, L, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(C, L, generator=g) * torch.exp(2 * torch.randn(C, 1, generator=g))     # channels of mixed scale
    x[:, ::97] *= 50.0                                                                     # and some large samples
    return x


def _guarded(n):
    buf = torch.full((n + 2 * GUARD,), float("nan"), device="cuda")
    return buf, buf[GUARD:GUARD + n]


def _seg(orig, new, xg, in_first, length, out, q0, q1):
    return dict(orig_rate=orig, new_rate=new, channels=xg.shape[0], in_=xg.data_ptr(), in_channel_stride=xg.stride(0),
                in_first=in_first, in_count=xg.shape[1], length=length, out=out.data_ptr(), out_first=q0,
                out_count=q1 - q0)


def _check(y, ref, bound, what):
    err = np.abs(y.double().cpu().numpy() - ref)
    assert np.all(err <= bound), (what, float((err / bound).max()))


def test_every_pair_against_float64_in_one_launch(eng):
    """Every rate pair to and from 48 kHz (and the identity) with C = 1, 2 and 6, all in one launch: whole signals
    (outputs at both edges), a range starting off a phase boundary read from a buffer that holds only its span, and a
    range of a signal whose length is not known yet.  Each output buffer has a guard band of NaN that stays untouched."""
    from sam_audio_b200.resample import input_span, outputs_ready, resampled_length
    rng = random.Random(0)
    segs, checks, keep = [], [], []
    for i, (orig, new) in enumerate(PAIRS):
        for C in (1, 2, 6):
            L = rng.randrange(3000, 9000)
            x = _signal(C, L, 100 * i + C)
            xg = x.cuda()
            keep.append(xg)
            N = resampled_length(L, orig, new)
            buf, out = _guarded(N)                                   # whole signal
            segs.append(_seg(orig, new, xg, 0, L, out, 0, N))
            checks.append((buf, out, x, orig, new, 0, N, L, "whole"))
            q0 = N // 3 + 1 + rng.randrange(0, 7)                    # off a phase boundary, span-sized buffer
            q1 = min(N, q0 + rng.randrange(1, 3000))
            i0, i1 = input_span(q0, q1, orig, new)
            i0, i1 = max(0, i0), min(L, i1)
            xs = xg[:, i0:i1].contiguous()
            keep.append(xs)
            buf, out = _guarded(q1 - q0)
            segs.append(_seg(orig, new, xs, i0, L, out, q0, q1))
            checks.append((buf, out, x, orig, new, q0, q1, L, "span"))
            a = L // 2                                               # length unknown: the outputs of a prefix
            qa = outputs_ready(a, orig, new)
            xp = xg[:, :a].contiguous()
            keep.append(xp)
            buf, out = _guarded(qa)
            segs.append(_seg(orig, new, xp, 0, -1, out, 0, qa))
            checks.append((buf, out, x, orig, new, 0, qa, L, "prefix"))
    eng.resample(segs)
    torch.cuda.synchronize()
    for buf, out, x, orig, new, q0, q1, L, what in checks:
        ref, bound = _reference(x, orig, new, q0, q1, L)
        _check(out, ref, bound, (orig, new, x.shape[0], what))
        assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + q1 - q0:]).all(), (orig, new, what)


@pytest.mark.parametrize("orig,new", [(44100, 48000), (48000, 16000), (8000, 48000), (48000, 8000), (44117, 48000),
                                      (48000, 11025)])
def test_any_segmentation_gives_the_same_bits(eng, orig, new):
    """The outputs of one signal split into random segments (one launch, or one launch per segment) equal the whole
    call's bits."""
    from sam_audio_b200.resample import input_span, resampled_length
    rng = random.Random(orig + new)
    L = 50_000
    xg = _signal(2, L, 7).cuda()
    N = resampled_length(L, orig, new)
    whole = torch.empty(N, device="cuda")
    eng.resample([_seg(orig, new, xg, 0, L, whole, 0, N)])
    for one_launch in (True, False):
        cuts = sorted(set([0, N] + [rng.randrange(1, N) for _ in range(rng.randrange(1, 40))]))
        got = torch.empty(N, device="cuda")
        segs, keep = [], []
        for q0, q1 in zip(cuts, cuts[1:]):
            i0, i1 = input_span(q0, q1, orig, new)
            i0, i1 = max(0, i0), min(L, i1)
            xs = xg[:, i0:i1].contiguous()
            keep.append(xs)
            segs.append(_seg(orig, new, xs, i0, L, got[q0:q1], q0, q1))
        if one_launch:
            eng.resample(segs)
        else:
            for s in segs:
                eng.resample([s])
        torch.cuda.synchronize()
        assert torch.equal(got, whole)


def test_model_resample(tiny_model):
    """SAMAudio.resample: [S] and [N, S] (each row its own signal, one launch), the identity returns its input."""
    x = _signal(3, 20_000, 3).cuda()
    y = tiny_model.resample(x, 16000, 48000)
    assert y.shape == (3, 60_000)
    for i in range(3):
        assert torch.equal(tiny_model.resample(x[i], 16000, 48000), y[i])
        ref, bound = _reference(x[i:i + 1].cpu(), 16000, 48000, 0, 60_000, 20_000)
        _check(y[i], ref, bound, i)
    assert tiny_model.resample(x, 48000, 48000) is x
    assert tiny_model.resample(y, 48000, 16000).shape == (3, 20_000)


# ---- streams ----
def _mean(x):
    """The channel mean as the kernel stages it: ascending sum, then one division."""
    m = x[0].clone()
    for c in range(1, x.shape[0]):
        m = m + x[c]
    return m / x.shape[0] if x.shape[0] > 1 else m


def _run(model, x, sizes, rate, ws=2.0, seed=0):
    s = model.stream(DESC, window_seconds=ws, seed=seed, sample_rate=rate)
    outs, i = [], 0
    for n in sizes:
        if i >= x.shape[-1]:
            break
        outs.append(s.push(x[..., i:i + n]))
        i += n
    if i < x.shape[-1]:
        outs.append(s.push(x[..., i:]))
    outs.append(s.flush())
    torch.cuda.synchronize()
    return torch.cat([o.target for o in outs]), torch.cat([o.residual for o in outs])


def _sizes(n, seed):
    rng = random.Random(seed)
    sizes, total = [], 0
    while total < n:
        s = rng.choice([1, 7, 159, 441, 1921, 4801, 16_001, 44_100, 100_003])
        sizes.append(s)
        total += s
    return sizes


def _composition(model, x, rate, ws=2.0, seed=0):
    """resample(out48, 48000, rate) of the 48 kHz stream pushed resample(mean_c(x), rate, 48000) whole."""
    x48 = model.resample(_mean(x), rate, 48000)
    t48, r48 = _run(model, x48, [x48.numel()], 48000, ws, seed)
    n48 = x48.numel()
    assert t48.numel() == math.ceil(n48 / 1920) * 1920
    return model.resample(t48, 48000, rate), model.resample(r48, 48000, rate)


def _audio(C, seconds, rate, seed):
    from sam_audio_b200.synthetic import synthetic_clip
    return torch.stack([synthetic_clip(seed + c, int(rate * seconds), sr=rate)[0] for c in range(C)]).cuda()


@pytest.mark.parametrize("which", ["tiny", "small"])
@pytest.mark.parametrize("rate,C", [(16000, 1), (44100, 2), (8000, 1)])
def test_stream_at_a_rate_equals_the_composition(request, which, rate, C):
    """Three random chunkings give identical bits, and they equal the composition of resample, the 48 kHz stream and
    resample back; the length is ceil(r' len48 / 48000') with len48 = ceil(n48 / hop) hop."""
    model = request.getfixturevalue("tiny_model" if which == "tiny" else "small_model")
    x = _audio(C, 9.3, rate, 5)
    if C == 1 and rate == 16000:
        x = x[0]                                                       # [S] as well as [1, S]
    n = x.shape[-1]
    runs = [_run(model, x, _sizes(n, k), rate) for k in range(3)]
    for t, r in runs[1:]:
        assert torch.equal(t, runs[0][0]) and torch.equal(r, runs[0][1])
    t, r = _composition(model, x.view(C, -1), rate)
    assert torch.equal(runs[0][0], t) and torch.equal(runs[0][1], r)
    n48 = math.ceil(48000 * n / rate)
    len48 = math.ceil(n48 / 1920) * 1920
    g = math.gcd(48000, rate)
    assert t.numel() == math.ceil((rate // g) * len48 / (48000 // g))


@pytest.fixture(scope="module")
def small_model(tiny_model):
    from sam_audio_b200.model import build_synthetic_model
    return build_synthetic_model("sam-audio-small", seed=0, device="cuda:0", weights_device="cuda:0")


def test_stereo_at_48k_is_the_mono_stream_of_its_mean(tiny_model):
    x = _audio(2, 7.1, 48000, 9)
    t, r = _run(tiny_model, x, _sizes(x.shape[1], 4), None)
    t1, r1 = _run(tiny_model, _mean(x), _sizes(x.shape[1], 5), None)
    assert torch.equal(t, t1) and torch.equal(r, r1)


def test_a_group_of_mixed_rates_equals_each_stream_alone(tiny_model, monkeypatch):
    """Four streams at 16 kHz mono, 44.1 kHz stereo, 8 kHz with six channels and 48 kHz mono in one group, pushed 0.5 s
    per tick with staggered starts: each equals the stream alone on the same pushes, and every tick makes at most two
    sab_resample calls (ingest and output)."""
    from sam_audio_b200 import _capi
    specs = [(16000, 1, 0), (44100, 2, 1), (8000, 6, 2), (48000, 1, 3)]
    wavs = [_audio(C, 6.0 + i, r, 20 + i) for i, (r, C, _) in enumerate(specs)]
    lib = _capi.lib()
    real = lib.sab_resample
    calls = []
    monkeypatch.setattr(lib, "sab_resample", lambda *a: calls.append(a[2]) or real(*a), raising=False)
    g = tiny_model.stream_group(window_seconds=2.0)
    streams, chunks, outs = [None] * 4, [[] for _ in specs], [[] for _ in specs]
    pos = [0] * 4
    tick = 0
    while any(p < w.shape[1] for p, w in zip(pos, wavs)):
        push = {}
        for i, ((rate, C, start), w) in enumerate(zip(specs, wavs)):
            if tick == start:
                streams[i] = g.open(DESC, seed=i, sample_rate=rate)
            if streams[i] is not None and pos[i] < w.shape[1]:
                c = w[:, pos[i]:pos[i] + rate // 2]
                pos[i] += c.shape[1]
                chunks[i].append(c)
                push[streams[i]] = c
        before = len(calls)
        res = g.push(push)
        assert len(calls) - before <= 2
        for i, s in enumerate(streams):
            if s in res:
                outs[i].append(res[s])
        tick += 1
    tails = g.close()
    torch.cuda.synchronize()
    monkeypatch.undo()
    for i, (rate, C, _) in enumerate(specs):
        outs[i].append(tails[streams[i]])
        t, r = torch.cat([o.target for o in outs[i]]), torch.cat([o.residual for o in outs[i]])
        s = tiny_model.stream(DESC, window_seconds=2.0, seed=i, sample_rate=rate)
        alone = [s.push(c) for c in chunks[i]] + [s.flush()]
        assert torch.equal(t, torch.cat([o.target for o in alone])), rate
        assert torch.equal(r, torch.cat([o.residual for o in alone])), rate


def test_48k_mono_makes_no_resample_call(tiny_model, monkeypatch):
    from sam_audio_b200 import _capi
    lib = _capi.lib()
    real = lib.sab_resample
    calls = []
    monkeypatch.setattr(lib, "sab_resample", lambda *a: calls.append(a[2]) or real(*a), raising=False)
    x = _audio(1, 5.0, 48000, 30)
    _run(tiny_model, x, [48000] * 6, None)
    _run(tiny_model, x[0], [30_000] * 9, 48000)
    assert calls == []
    _run(tiny_model, _audio(1, 3.0, 16000, 31), [16000] * 4, 16000)
    assert calls


def test_memory_is_bounded_at_16k(tiny_model):
    """1 s pushes at 16 kHz and W = 50: the engine's workspace and the allocator's peak after 20 windows equal those
    after 3."""
    x = _audio(1, 40.0, 16000, 40)[0]
    s = tiny_model.stream(DESC, window_seconds=2.0, sample_rate=16000)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    at = {}
    for i in range(0, x.numel(), 16000):
        s.push(x[i:i + 16000])
        if s.windows_solved in (3, 20) and s.windows_solved not in at:
            torch.cuda.synchronize()
            at[s.windows_solved] = (s.workspace_bytes(), torch.cuda.max_memory_allocated())
    s.flush()
    assert set(at) == {3, 20}
    assert at[20] == at[3]


def test_stream_channel_count_is_fixed_by_the_first_push(tiny_model):
    s = tiny_model.stream(DESC, window_seconds=2.0, sample_rate=16000)
    s.push(torch.zeros(2, 1000, device="cuda"))
    with pytest.raises(ValueError, match="has 2 channel"):
        s.push(torch.zeros(1000, device="cuda"))
    assert s.flush().target.numel() == math.ceil(math.ceil(1000 * 3 / 1920) * 1920 / 3)
