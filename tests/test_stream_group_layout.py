"""CPU: the host rules of stream groups (SAMAudio.stream_group): the item buckets of planned calls, the grouped solves
of a tick against the single-stream rules, and the argument checks of a tick."""
import math
import random
from types import SimpleNamespace

import pytest
import torch

from sam_audio_b200.stream import check_tick
from sam_audio_b200.windows import (stream_bucket, stream_buckets, stream_emit_end, stream_final_frames,
                                    stream_flush_rows, stream_frames_available, stream_group_capacity, stream_tick_groups,
                                    stream_window_starts, stream_windows_ready, window_groups)

HOP, HALO_ENC, HALO_DEC = 1920, 6, 8          # the standard codec rates (sab_codec_tiling reports these halos)


@pytest.mark.parametrize("capacity", [1, 2, 3, 4, 5, 7, 8, 9, 64, 400, 2000])
def test_bucket_rule(capacity):
    """The smallest power of two >= n, capped at the capacity; live items in their own slots, filler slots pointing at
    live items; a call of more items than the capacity is refused."""
    buckets = stream_buckets(capacity)
    assert buckets[-1] == capacity and buckets == sorted(set(buckets))
    assert all(b == 1 << i for i, b in enumerate(buckets[:-1]))
    for n in range(1, capacity + 1):
        slots = stream_bucket(n, capacity)
        assert len(slots) == min(capacity, 1 << math.ceil(math.log2(n))) and len(slots) in buckets
        assert slots[:n] == list(range(n))
        assert all(0 <= s < n for s in slots)
    for n in (0, capacity + 1):
        with pytest.raises(ValueError):
            stream_bucket(n, capacity)


def test_flush_reuses_resident_buckets():
    """A flush tick's solves are grouped by at most the largest resident bucket of windows and each runs at the smallest
    resident bucket that holds it, so ending many streams at once plans no larger bucket; with nothing resident (or no
    resident bucket large enough) the power-of-two rule applies."""
    W, cap = 250, 400
    for resident in ({8}, {4, 8}, {1, 2, 16}):
        rows = stream_flush_rows(100_000, W, resident)
        assert rows == max(resident) * W
        for n_windows in (1, 3, 64, 101):
            for g0, g1 in window_groups(n_windows, 1, W, rows):
                slots = stream_bucket(g1 - g0, cap, resident)
                assert len(slots) in resident and len(slots) == min(b for b in resident if b >= g1 - g0)
                assert slots[:g1 - g0] == list(range(g1 - g0)) and all(0 <= x < g1 - g0 for x in slots)
    assert stream_flush_rows(100_000, W, set()) == 100_000
    assert len(stream_bucket(5, cap, set())) == 8 and len(stream_bucket(5, cap, {4})) == 8
    assert len(stream_bucket(3, cap, {4, 64})) == 4


def test_capacity_is_one_grouped_solve():
    for W in (8, 50, 250, 10000):
        for budget in (1, W, 3 * W + 1, 100_000):
            per = stream_group_capacity(W, budget)
            assert per == max(1, budget // W)
            assert all(g1 - g0 <= per for g0, g1 in window_groups(1000, 1, W, budget))


class _Sim:
    """The counters of one stream advanced as StreamGroup advances them: the windows of a tick come from
    stream_tick_groups, a group's last range of a stream decides its flush-time pad, final frames and emission."""

    def __init__(self, W):
        self.W, self.n, self.solved, self.final, self.emitted, self.n_final = W, 0, 0, 0, 0, None

    def due(self, flushed):
        if flushed:
            self.n_final = -(-self.n // HOP)
            return len(stream_window_starts(self.n_final, self.W)) if self.n else self.solved
        return stream_windows_ready(stream_frames_available(self.n, HOP, HALO_ENC), self.W)


def _run_tick(sims, pushes, flushed, W, budget):
    for s, x in pushes.items():
        s.n += x
    due = [(s, s.solved, s.due(flushed)) for s in pushes]
    groups = stream_tick_groups(due, W, budget)
    cap = stream_group_capacity(W, budget)
    ranges = {s: [] for s in pushes}
    for grp in groups:
        assert 1 <= sum(w.kb - w.ka for w in grp) <= cap
        assert len({id(w.key) for w in grp}) == len(grp)         # one range per stream and group
        for w in grp:
            ranges[w.key].append((w.ka, w.kb))
            fl = flushed and w.last
            assert w.last == (w.kb == dict((id(k), e) for k, _, e in due)[id(w.key)])
            s = w.key
            assert w.ka == s.solved                              # in order, no window twice
            s.solved = w.kb
            s.final = stream_final_frames(w.kb, W, s.n_final if fl else -1)
            s.emitted = max(s.emitted, stream_emit_end(s.final, HALO_DEC, fl))
    # a flat list of all windows, grouped as window_groups groups it
    assert [sum(w.kb - w.ka for w in g) for g in groups] == \
        [g1 - g0 for g0, g1 in window_groups(sum(e - k for _, k, e in due), 1, W, budget)]
    for s, k0, k_end in due:
        got = [k for a, b in ranges[s] for k in range(a, b)]
        assert got == list(range(k0, k_end))


def _check_single_stream_rules(s, W, flushed):
    if flushed:
        if s.n:
            assert s.solved == len(stream_window_starts(s.n_final, W))
            assert s.final == s.emitted == s.n_final
        return
    assert s.solved == stream_windows_ready(stream_frames_available(s.n, HOP, HALO_ENC), W)
    assert s.final == stream_final_frames(s.solved, W)
    if s.solved:
        assert s.emitted == stream_emit_end(s.final, HALO_DEC, False)


def _chunk(rng):
    return rng.choice([1, 1, 7, HOP - 1, HOP + 1, 4801, 48000, 48000, 48000, 96_001, 500_000])


@pytest.mark.parametrize("W,budget", [(50, 100_000), (50, 150), (250, 100_000), (250, 250), (8, 24)])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_tick_schedule_matches_single_stream_rules(W, budget, seed):
    """Staggered starts, joins and leaves, pushes of 1 sample and of non-multiples of the hop, ticks that push any
    subset of the open streams: after every tick each stream's windows, final frames and emitted frames are those the
    single-stream rules give for the samples it has received, and its windows arrive in order, each once; a stream
    advanced alone through the same pushes passes through the same counters."""
    rng = random.Random(seed)
    group, solo, history = [], {}, {}
    for tick in range(60):
        if tick < 40 and (not group or rng.random() < 0.2):
            s = _Sim(W)
            group.append(s)
            solo[s] = _Sim(W)
            history[s] = []
        if not group:
            continue
        pushing = {s: _chunk(rng) for s in group if rng.random() < 0.7}
        if pushing:
            _run_tick(group, pushing, False, W, budget)
            for s, x in pushing.items():
                _run_tick([solo[s]], {solo[s]: x}, False, W, budget)
                _check_single_stream_rules(s, W, False)
                assert (s.solved, s.final, s.emitted) == (solo[s].solved, solo[s].final, solo[s].emitted)
        leaving = [s for s in group if rng.random() < 0.08 or tick == 59]
        if leaving:
            _run_tick(group, {s: 0 for s in leaving}, True, W, budget)
            for s in leaving:
                _run_tick([solo[s]], {solo[s]: 0}, True, W, budget)
                _check_single_stream_rules(s, W, True)
                assert (s.solved, s.final, s.emitted) == (solo[s].solved, solo[s].final, solo[s].emitted)
                group.remove(s)
    assert not group


def test_one_stream_many_windows_in_one_tick_respects_the_group_size():
    """A single push that makes many windows ready is solved in groups of at most the capacity, in order."""
    W, budget = 50, 3 * 50
    s = _Sim(W)
    _run_tick([s], {s: 200 * W * HOP}, False, W, budget)
    _check_single_stream_rules(s, W, False)
    assert s.solved > 3


def _fake_group(W=250):
    return SimpleNamespace(W=W)


def _fake_stream(group, W=None, closed=False):
    return SimpleNamespace(group=group, W=group.W if W is None else W, closed=closed)


def test_tick_argument_checks():
    g, other = _fake_group(), _fake_group()
    a, b = _fake_stream(g), _fake_stream(g)
    check_tick(g, [a, b])
    check_tick(g, [])
    with pytest.raises(RuntimeError, match="closed"):
        check_tick(g, [a, _fake_stream(g, closed=True)])
    with pytest.raises(ValueError, match="another group"):
        check_tick(g, [a, _fake_stream(other)])
    with pytest.raises(ValueError, match="another group"):
        check_tick(g, [object()])
    with pytest.raises(ValueError, match="window of 50 frames in a group of 250"):
        check_tick(g, [_fake_stream(g, W=50)])
    with pytest.raises(ValueError, match="twice"):
        check_tick(g, [a, a])


@pytest.fixture(scope="module")
def cpu_model():
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    cfg = stand_in_config("sam-audio-tiny", transformer={"max_positions": 320})
    return SAMAudio(cfg, text_encoder=SyntheticTextEncoder(cfg.text_encoder.dim))


@pytest.mark.parametrize("kw,why", [(dict(reranking_candidates=2), "one candidate"),
                                    (dict(anchors=[["+", 1.0, 2.0]]), "time base"),
                                    (dict(masked_video=torch.zeros(4, 3, 8, 8)), "time base"),
                                    (dict(ode_opt={"method": "dopri5"}), "fixed-grid")])
def test_stream_group_refuses_what_stream_refuses(cpu_model, kw, why):
    with pytest.raises(NotImplementedError, match=why):
        cpu_model.stream_group(**kw)


def test_stream_group_window_is_checked(cpu_model):
    with pytest.raises(ValueError, match="8 <= W <= 320"):
        cpu_model.stream_group(window_seconds=20.0)
