"""CPU: the window layout of batches longer than the position table (sam_audio_b200.windows) and the fp64 blend of the
windowed oracle."""
import math

import pytest
import torch

from sam_audio_b200.windows import (clip_window_starts, window_groups, window_layout, window_ramp,
                                    DEFAULT_WINDOW_ROWS)

TW = 10000
CASES = [(TW, 1), (TW + 1, 2), (15000, 2), (18750, 2), (18751, 3), (45000, 5), (320, 1), (750, 1), (123457, 14)]


@pytest.mark.parametrize("Tw", [320, 1000, TW])
@pytest.mark.parametrize("n", [1, 100, 319, 320, 321, 559, 560, 561, 750, 1500, 9999, 10000, 10001, 17500, 45000,
                               150000])
def test_layout_covers_overlaps_and_is_minimal(n, Tw):
    O = window_ramp(Tw)
    assert O == Tw // 8
    starts = clip_window_starts(n, Tw)
    if n <= Tw:
        assert starts == [0]
        return
    W = len(starts)
    assert starts[0] == 0 and starts[-1] + Tw == n                      # flush with the clip at both ends
    assert all(0 <= s and s + Tw <= n for s in starts)                  # every window lies inside [0, n)
    assert starts == sorted(starts)
    covered = torch.zeros(n, dtype=torch.bool)
    for s in starts:
        covered[s:s + Tw] = True
    assert bool(covered.all())
    assert all(a + Tw - b >= O for a, b in zip(starts, starts[1:]))     # adjacent overlaps >= O
    # minimal for the stride Tw - O: W - 1 windows cannot reach n with overlaps >= O
    assert (W - 2) * (Tw - O) + Tw < n
    assert W == 1 + math.ceil((n - Tw) / (Tw - O))
    assert starts == [k * (n - Tw) // (W - 1) for k in range(W)]


@pytest.mark.parametrize("n,W", CASES)
def test_window_counts(n, W):
    assert len(clip_window_starts(n, TW)) == W


def test_one_frame_past_the_table_gives_two_windows():
    assert clip_window_starts(TW + 1, TW) == [0, 1]


def test_ragged_batch_gives_per_clip_counts_in_clip_order():
    sizes = torch.tensor([750.0, 250.0, 1500.0, 320.0])
    wins = window_layout(sizes, 320)
    per = [clip_window_starts(int(n), 320) for n in sizes]
    assert [len(p) for p in per] == [3, 1, 6, 1]
    assert [w.clip for w in wins] == [0] * 3 + [1] + [2] * 6 + [3]
    assert [w.start for w in wins] == [s for p in per for s in p]
    for b in range(4):
        mine = [w for w in wins if w.clip == b]
        assert mine[0].first and mine[-1].last
        assert not any(w.first for w in mine[1:]) and not any(w.last for w in mine[:-1])


def test_groups_hold_whole_windows_within_budget():
    assert window_groups(7, 2, 320, 3 * 2 * 320) == [(0, 3), (3, 6), (6, 7)]
    assert window_groups(7, 2, 320, 1) == [(i, i + 1) for i in range(7)]     # at least one window per group
    assert window_groups(5, 1, TW, DEFAULT_WINDOW_ROWS) == [(0, 5)]


def test_window_rows_budget_follows_the_environment(monkeypatch):
    from sam_audio_b200.windows import window_rows_budget
    monkeypatch.delenv("SAB_WINDOW_ROWS", raising=False)
    assert window_rows_budget() == DEFAULT_WINDOW_ROWS
    monkeypatch.setenv("SAB_WINDOW_ROWS", "1")
    assert window_rows_budget() == 1


@pytest.mark.parametrize("c", [1, 2])
def test_oracle_blend_reproduces_a_latent_from_its_windows(c):
    from _oracle_windowed import blend_fp64
    sizes, Tw, T = [750, 250, 601], 320, 750
    wins = window_layout(sizes, Tw)
    lat = torch.randn(len(sizes) * c, T, 256, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    cut = torch.stack([lat[w.clip * c + k, w.start:w.start + Tw] for w in wins for k in range(c)])
    out = blend_fp64(cut, wins, c, len(sizes), T, window_ramp(Tw))
    for b, n in enumerate(sizes):
        covered = slice(0, max(n, Tw))
        rows = slice(b * c, (b + 1) * c)
        assert torch.allclose(out[rows, covered], lat[rows, covered], rtol=1e-12, atol=1e-12)
        assert bool((out[rows, max(n, Tw):] == 0).all())                     # uncovered pad frames are 0
