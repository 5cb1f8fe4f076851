"""CPU: the resampler's table (sab_resample_taps) against torchaudio and against the formula, its index rules
(sam_audio_b200.resample) against a brute-force enumeration of tap indices, and the argument checks of sab_resample,
SAMAudio.resample() and streams at other rates, none of which touch CUDA."""
import ctypes
import math
import random

import numpy as np
import pytest
import torch

RATES = [8000, 11025, 16000, 22050, 32000, 44100, 96000, 192000]
PAIRS = [(r, 48000) for r in RATES] + [(48000, r) for r in RATES]


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    return _capi.lib()


def _apply(x, orig, new, K, lo, w):
    """The table applied in float64: y[q] = sum_k w[j][k] x[m o + lo[j] + k], zero outside [0, len(x))."""
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    N = -(-n * len(x) // o)
    q = np.arange(N)
    j = q % n
    idx = ((q // n) * o + lo[j])[:, None] + np.arange(K)[None, :]
    valid = (idx >= 0) & (idx < len(x))
    xs = np.where(valid, x[np.clip(idx, 0, len(x) - 1)], 0.0)
    return (w[j].astype(np.float64) * xs).sum(1)


@pytest.mark.parametrize("orig,new", PAIRS)
def test_table_matches_torchaudio(lib, orig, new):
    """Within 1e-6 max|x| of torchaudio.functional.resample on float64 noise, with the same length."""
    import torchaudio
    from sam_audio_b200 import _capi
    K, lo, w = _capi.resample_taps(orig, new)
    x = np.random.default_rng(orig + new).standard_normal(2003)
    ours = _apply(x, orig, new, K, lo, w)
    ref = torchaudio.functional.resample(torch.from_numpy(x), orig, new).numpy()
    assert ours.shape == ref.shape
    if orig == new:
        assert K == 1 and np.array_equal(ours, x)
    assert np.abs(ours - ref).max() <= 1e-6 * np.abs(x).max()


def test_table_sizes(lib):
    """K = 15 for every upsampling to 48 kHz and for 48k -> 44.1k, 29 for 48k -> 22.05k, 39 for 48k -> 16k, 75 for
    48k -> 8k; the identity has one tap of weight 1."""
    from sam_audio_b200 import _capi
    for r in RATES:
        if r < 48000:
            assert _capi.resample_taps(r, 48000)[0] == 15
    for r, K in ((44100, 15), (22050, 29), (16000, 39), (8000, 75)):
        assert _capi.resample_taps(48000, r)[0] == K
    K, lo, w = _capi.resample_taps(48000, 48000)
    assert K == 1 and lo.tolist() == [0] and w.tolist() == [[1.0]]


def _formula(orig, new):
    """An independent float64 evaluation of the design: lo from exact fractions, weights from the formula."""
    from fractions import Fraction
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    base = Fraction(99, 100) * min(o, n)
    R = 6 * Fraction(o) / base
    K = 2 * math.ceil(R) + 1
    lo = np.array([math.ceil(Fraction(j * o, n) - R) for j in range(n)], np.int64)
    # (lo + k) / o - j / n over the common denominator o n: exact in the numerator, one rounding in the division
    t = ((lo[:, None] + np.arange(K)[None, :]) * n - np.arange(n)[:, None] * o) / (o * n) * float(base)
    t = np.clip(t, -6.0, 6.0)
    w = np.sinc(t) * np.cos(np.pi * t / 12) ** 2 * float(base) / o
    return K, lo, w, o, n, float(base)


@pytest.mark.parametrize("orig,new", [(44117, 48000), (48000, 44117), (44100, 48000), (48000, 8000)])
def test_table_matches_the_formula(lib, orig, new):
    """For a coprime pair (whose dense torchaudio kernel would take 17 GB) and two common ones: the same K and lo, the
    weights within one fp32 rounding, and no tap left out: the indices just before and after each phase's window have
    |t| >= 6, where the window is zero."""
    from sam_audio_b200 import _capi
    K, lo, w = _capi.resample_taps(orig, new)
    K2, lo2, w2, o, n, base = _formula(orig, new)
    assert K == K2 and np.array_equal(lo, lo2)
    # one fp32 rounding (and fp32's smallest subnormal where the window's tail underflows)
    assert np.all(np.abs(w - w2) <= 2.0 ** -24 * np.abs(w2) + 2.0 ** -149)
    j = np.arange(n)
    assert np.all(((lo - 1) / o - j / n) * base <= -6.0)
    assert np.all(((lo + K) / o - j / n) * base >= 6.0)


def _brute(orig, new, q_max):
    """Every tap index of outputs [0, q_max), enumerated from the table."""
    from sam_audio_b200 import _capi
    g = math.gcd(orig, new)
    o, n = orig // g, new // g
    K, lo, _ = _capi.resample_taps(orig, new)
    return [[(q // n) * o + int(lo[q % n]) + k for k in range(K)] for q in range(q_max)]


@pytest.mark.parametrize("orig,new", [(16000, 48000), (44100, 48000), (48000, 44100), (48000, 8000), (48000, 48000),
                                      (44117, 48000), (192000, 48000)])
def test_index_rules_match_brute_force(lib, orig, new):
    from sam_audio_b200.resample import input_span, outputs_ready, resampled_length
    rng = random.Random(orig * 7 + new)
    q_max = math.ceil(1600 * new / orig) + 50                # past every output ready from 1500 samples
    tap = _brute(orig, new, q_max)
    for _ in range(200):
        a = rng.randrange(0, 1500)
        ready = [max(t) < a for t in tap]                   # an output needs every tap index below a
        k = outputs_ready(a, orig, new)
        assert k < q_max and all(ready[:k]) and not any(ready[k:])
        L = rng.randrange(1, 1500)
        assert outputs_ready(L, orig, new, length=L) == resampled_length(L, orig, new) == math.ceil(new * L / orig)
        q0 = rng.randrange(0, q_max // 2)
        q1 = q0 + rng.randrange(1, q_max // 2)
        span = [i for t in tap[q0:q1] for i in t]
        assert input_span(q0, q1, orig, new) == (min(span), max(span) + 1)


_FAKE = 1 << 20     # a non-null address: the checks run before anything is dereferenced


def _seg(**kw):
    from sam_audio_b200 import _capi
    d = dict(orig_rate=16000, new_rate=48000, channels=1, in_=_FAKE, in_channel_stride=1000, in_first=0, in_count=1000,
             length=1000, out=_FAKE, out_first=0, out_count=3000)
    d.update(kw)
    return _capi.SabResampleSeg(**d)


def _error(lib, *segs):
    from sam_audio_b200 import _capi
    arr = _capi.resample_segments(list(segs))
    rc = lib.sab_resample(None, arr, len(segs), None)
    assert rc != 0
    return lib.sab_last_error().decode()


@pytest.mark.parametrize("fields,message", [
    (dict(orig_rate=7999), "rates 7999 -> 48000"),
    (dict(new_rate=192001), "rates 16000 -> 192001"),
    (dict(channels=0), "channels=0 outside 1..8"),
    (dict(channels=9, in_channel_stride=1000), "channels=9 outside 1..8"),
    (dict(channels=2, in_channel_stride=999), "channel stride 999 < in_count 1000"),
    (dict(out_count=-1), "negative count"),
    (dict(in_count=-5), "negative count"),
    (dict(out_count=3001), "past the 3000 of a 1000-sample signal"),
    (dict(in_first=1), "read input samples [0, 1000), the buffer holds [1, 1001)"),
    (dict(in_count=999, length=-1, out_count=2980), "read input samples [0, 1002), the buffer holds [0, 999)"),
    (dict(length=-1), "read input samples [0, 1009)"),          # unknown length: the taps past 999 must be there too
    (dict(out=None), "null output"),
    (dict(in_=None), "null input"),
])
def test_resample_arguments_are_checked_on_the_host(lib, fields, message):
    """Host-only: each rule fails with its message before any CUDA call (the engine is NULL, so a segment list that
    passed the rules would fail at 'null engine')."""
    err = _error(lib, _seg(**fields))
    assert message in err, err


def test_resample_rules_pass_then_the_engine_is_needed(lib):
    for segs in ([_seg()], [_seg(length=-1, out_count=2970)], [_seg(out_first=1, out_count=5)],
                 [_seg(in_first=400, in_count=300, out_first=1500, out_count=10)], [_seg(), _seg(out_count=0, out=None)],
                 [_seg(channels=8, in_channel_stride=1000, orig_rate=48000, new_rate=48000, out_count=1000)]):
        assert "null engine" in _error(lib, *segs)


def test_resample_struct_bytes_rejected(lib):
    from sam_audio_b200 import _capi
    assert ctypes.sizeof(_capi.SabResampleSeg) % 8 == 0
    for wrong in (ctypes.sizeof(_capi.SabResampleSeg) - 8, 0):
        err = _error(lib, _seg(), _seg(struct_bytes=wrong))
        assert "struct_bytes" in err and "header and binding differ" in err, err


def test_resample_taps_checks(lib):
    K = ctypes.c_int()
    assert lib.sab_resample_taps(48000, 7000, 0, ctypes.byref(K), None, None) != 0
    assert b"[8000, 192000]" in lib.sab_last_error()
    w = np.zeros(10, np.float32)
    assert lib.sab_resample_taps(48000, 16000, w.size, ctypes.byref(K), None, w.ctypes.data) != 0
    assert b"tap capacity 10 < 39" in lib.sab_last_error()


@pytest.fixture(scope="module")
def cpu_model():
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    cfg = stand_in_config("sam-audio-tiny")
    return SAMAudio(cfg, text_encoder=SyntheticTextEncoder(cfg.text_encoder.dim))


@pytest.mark.parametrize("rate", [7999, 192001, 16000.5, "16000", True])
def test_stream_rate_is_checked(cpu_model, rate):
    with pytest.raises((ValueError, TypeError), match="sample_rate"):
        cpu_model.stream("rain", sample_rate=rate)


def test_pushed_shapes_are_checked():
    from sam_audio_b200.stream import _samples
    assert _samples(torch.zeros(5)).shape == (1, 5)
    assert _samples(torch.zeros(1, 5)).shape == (1, 5)
    assert _samples(torch.zeros(8, 5)).shape == (8, 5)
    assert _samples(torch.zeros(2, 5), channels=2).shape == (2, 5)
    for bad in (torch.zeros(0), torch.zeros(9, 5), torch.zeros(2, 0), torch.zeros(1, 2, 3), torch.zeros(())):
        with pytest.raises(ValueError, match=r"\[C, S\]"):
            _samples(bad)
    with pytest.raises(ValueError, match="has 2 channel"):
        _samples(torch.zeros(1, 5), channels=2)
    with pytest.raises(TypeError):
        _samples([0.0, 1.0])


@pytest.mark.parametrize("args,message", [
    ((torch.zeros(10), 16000, 7000), "new_sr=7000"),
    ((torch.zeros(10), 7000, 48000), "orig_sr=7000"),
    ((torch.zeros(10), 16000, 44100), "one side must be the model's rate"),
    ((torch.zeros(2, 3, 10), 16000, 48000), r"\[S\] or \[N, S\]"),
    ((torch.zeros(0), 16000, 48000), r"\[S\] or \[N, S\]"),
    ((torch.zeros(10), 16000, 48000), "CUDA device"),
    ((torch.zeros(10, dtype=torch.float64), 48000, 48000), "fp32"),
])
def test_model_resample_arguments(cpu_model, args, message):
    with pytest.raises(ValueError, match=message):
        cpu_model.resample(*args)
