"""CPU: the index rules of the multichannel stems (sam_audio_b200.channels) against a brute-force enumeration of the
frames each sample reads, over random push sequences and their flush; the latency bound; and the argument checks of
sab_spread_channels, SAMAudio.spread_channels() and keep_channels, none of which touch CUDA."""
import ctypes
import random

import pytest
import torch

from sam_audio_b200.channels import HOP, LATENCY, N, frame_span, frames_of, input_span, keep_from, spread_ready


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    return _capi.lib()


def _frame_known(j, received, length):
    """Every sample frame j reads (>= 0) is below `received` or at / past the known `length`."""
    i0, i1 = frame_span(j)
    return all(i < received or (length is not None and i >= length) for i in range(max(0, i0), i1))


def _brute_ready(tr_received, x_received, tr_length, x_length, limit):
    """The longest prefix of outputs (below tr_length when known, below `limit` otherwise) whose four frames are all
    computable from both inputs, sample by sample (each frame's verdict enumerated once)."""
    known = {}

    def ok(j):
        if j not in known:
            known[j] = _frame_known(j, tr_received, tr_length) and _frame_known(j, x_received, x_length)
        return known[j]
    s = 0
    end = limit if tr_length is None else tr_length
    while s < end and all(ok(j) for j in range(*frames_of(s))):
        s += 1
    return s


def test_frames_cover_each_sample_four_times():
    for s in list(range(0, 3 * HOP)) + [10_000, 10_239, 10_240]:
        js = [j for j in range(0, s // HOP + 10) if frame_span(j)[0] <= s < frame_span(j)[1]]
        assert js == list(range(*frames_of(s))) and len(js) == 4 and frame_span(0) == (-3 * HOP, HOP)
    assert N == 4 * HOP and LATENCY == N


def test_readiness_matches_brute_force_over_random_pushes():
    """A stream's inputs grow as a keep-channels stream feeds them: the channels by pushes of any size, the mono stems
    in whole codec hops (1920 samples) lagging behind; at the flush both lengths become known (stems ceil(n / 1920)
    1920, channels n).  At every step the rule equals the brute force, is a multiple of a before the flush, never
    shrinks, and no output waits for more than LATENCY samples of both inputs past it."""
    rng = random.Random(0)
    for trial in range(25):
        x_rec = tr_rec = 0
        produced = 0
        for _ in range(rng.randrange(1, 12)):
            x_rec += rng.choice([1, 7, 300, 511, 512, 1920, 4801])
            tr_rec = max(tr_rec, rng.randrange(0, x_rec // 1920 + 1) * 1920)
            r = spread_ready(tr_rec, x_rec)
            assert r == _brute_ready(tr_rec, x_rec, None, None, min(tr_rec, x_rec) + N), (trial, tr_rec, x_rec)
            assert r % HOP == 0 and r >= produced
            assert r > min(tr_rec, x_rec) - LATENCY
            produced = r
        tr_len = -(-x_rec // 1920) * 1920
        r = spread_ready(tr_len, x_rec, tr_len, x_rec)
        assert r == tr_len == _brute_ready(tr_len, x_rec, tr_len, x_rec, 0) and r >= produced


@pytest.mark.parametrize("tr_len,x_len", [(None, 5000), (6000, None)])
def test_readiness_with_one_length_known(tr_len, x_len):
    for tr_rec in range(0, 6001, 750):
        for x_rec in (0, 1000, 2500, 5000):
            if (tr_len is not None and tr_rec != tr_len) or (x_len is not None and x_rec != x_len):
                continue
            limit = min([v for v, L in ((tr_rec, tr_len), (x_rec, x_len)) if L is None]) + N
            assert spread_ready(tr_rec, x_rec, tr_len, x_len) == _brute_ready(tr_rec, x_rec, tr_len, x_len, limit)


def test_input_span_and_trim_match_brute_force():
    rng = random.Random(1)
    for _ in range(300):
        s0 = rng.randrange(0, 6000)
        s1 = s0 + rng.randrange(1, 3000)
        spans = [frame_span(j) for j in {j for s in range(s0, s1) for j in range(*frames_of(s))}]
        assert input_span(s0, s1) == (min(a for a, _ in spans), max(b for _, b in spans))
        later = [i for j in range(*frames_of(s0)) for i in range(*frame_span(j))]
        assert keep_from(s0) == max(0, min(later))


_FAKE = 1 << 20     # a non-null address: the checks run before anything is dereferenced


def _seg(**kw):
    from sam_audio_b200 import _capi
    d = dict(channels=2, target=_FAKE, residual=_FAKE, tr_first=0, tr_count=4000, tr_length=4000, mix=_FAKE,
             mix_channel_stride=4000, mix_first=0, mix_count=3500, mix_length=3500, out_target=_FAKE,
             out_residual=_FAKE, out_channel_stride=4000, out_first=0, out_count=4000)
    d.update(kw)
    return _capi.SabSpreadSeg(**d)


def _error(lib, *segs):
    from sam_audio_b200 import _capi
    arr = _capi.spread_segments(list(segs))
    rc = lib.sab_spread_channels(None, arr, len(segs), None)
    assert rc != 0
    return lib.sab_last_error().decode()


@pytest.mark.parametrize("fields,message", [
    (dict(channels=0), "channels=0 outside 1..8"),
    (dict(channels=9), "channels=9 outside 1..8"),
    (dict(out_count=-1), "negative count"),
    (dict(tr_length=-2), "negative count"),
    (dict(mix_channel_stride=3000), "mix channel stride 3000 < mix_count 3500"),
    (dict(out_channel_stride=100), "output channel stride 100 < out_count 4000"),
    (dict(mix_length=4001, mix_count=4001, mix_channel_stride=4001), "longer than its 4000-sample stems"),
    (dict(out_count=4001, out_channel_stride=4001), "past the end of 4000-sample stems"),
    (dict(out_residual=None), "null output"),
    (dict(tr_first=1, tr_count=3999), "read stem samples [0, 4000), the buffers hold [1, 4000)"),
    (dict(tr_length=-1, out_count=2049), "read stem samples [0, 4096), the buffers hold [0, 4000)"),
    (dict(mix_count=3000, mix_channel_stride=3000), "read mixture samples [0, 3500), the buffer holds [0, 3000)"),
    (dict(mix_length=-1, mix_count=3000, mix_channel_stride=3000, out_first=1024, out_count=10),
     "read mixture samples [0, 3072), the buffer holds [0, 3000)"),
    (dict(target=None), "null stems"),
    (dict(mix=None), "null mixture"),
])
def test_spread_arguments_are_checked_on_the_host(lib, fields, message):
    """Host-only: each rule fails with its message before any CUDA call (the engine is NULL, so a segment list that
    passed the rules would fail at 'null engine')."""
    err = _error(lib, _seg(**fields))
    assert message in err, err


def test_spread_rules_pass_then_the_engine_is_needed(lib):
    for segs in ([_seg()], [_seg(channels=8, mix_channel_stride=3500)], [_seg(tr_length=-1, out_count=1536)],
                 [_seg(tr_first=1024, tr_count=2976, out_first=2560, out_count=1440, mix_first=1024, mix_count=2476)],
                 [_seg(mix_length=-1, mix_count=3584, mix_channel_stride=3584, out_count=1024)],
                 [_seg(), _seg(out_count=0, out_target=None, out_residual=None)],
                 [_seg(mix=None, mix_count=0, mix_length=0)]):
        assert "null engine" in _error(lib, *segs)


def test_spread_struct_bytes_rejected(lib):
    from sam_audio_b200 import _capi
    assert ctypes.sizeof(_capi.SabSpreadSeg) % 8 == 0
    for wrong in (ctypes.sizeof(_capi.SabSpreadSeg) - 8, 0):
        err = _error(lib, _seg(), _seg(struct_bytes=wrong))
        assert "struct_bytes" in err and "header and binding differ" in err, err


@pytest.fixture(scope="module")
def cpu_model():
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    cfg = stand_in_config("sam-audio-tiny")
    return SAMAudio(cfg, text_encoder=SyntheticTextEncoder(cfg.text_encoder.dim))


@pytest.mark.parametrize("value", [1, 0, "yes", None])
def test_keep_channels_is_checked(cpu_model, value):
    with pytest.raises(TypeError, match="keep_channels"):
        cpu_model.stream("rain", keep_channels=value)


def test_keep_channels_is_checked_by_open_and_submit():
    from sam_audio_b200.stream import StreamGroup
    group = StreamGroup.__new__(StreamGroup)            # the checks run before any engine state is read
    group.closed = False
    with pytest.raises(TypeError, match="keep_channels"):
        group.open("rain", keep_channels=1)
    with pytest.raises(TypeError, match="keep_channels"):
        group.submit(torch.zeros(2, 100), "rain", keep_channels="yes")


@pytest.mark.parametrize("args,message", [
    ((torch.zeros(10), torch.zeros(10), torch.zeros(2, 10, dtype=torch.float64)), "fp32"),
    ((torch.zeros(10), torch.zeros(10), torch.zeros(2, 10)), "CUDA device"),
    ((torch.zeros(10), torch.zeros(9), torch.zeros(2, 9)), r"one length \[S'\]"),
    ((torch.zeros(1, 10), torch.zeros(1, 10), torch.zeros(2, 10)), r"one length \[S'\]"),
    ((torch.zeros(0), torch.zeros(0), torch.zeros(1, 0)), r"one length \[S'\]"),
    ((torch.zeros(10), torch.zeros(10), torch.zeros(10)), r"mixture \[C, S\]"),
    ((torch.zeros(10), torch.zeros(10), torch.zeros(9, 10)), r"mixture \[C, S\]"),
    ((torch.zeros(10), torch.zeros(10), torch.zeros(2, 11)), r"S <= S' = 10"),
    ((torch.zeros(10), torch.zeros(10), torch.zeros(2, 0)), r"mixture \[C, S\]"),
    ((torch.zeros(10), torch.zeros(10), [[0.0] * 10]), "takes tensors"),
])
def test_spread_channels_arguments(cpu_model, args, message):
    with pytest.raises(ValueError, match=message):
        cpu_model.spread_channels(*args)
