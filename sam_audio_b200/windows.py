"""Windowed solving of batches longer than the model's position table (DESIGN.md section 3).

The DiT's RoPE table ends at ``transformer.max_positions`` frames (reference rope.py:152), so ``SAMAudio.separate()``
solves a longer batch as overlapping windows of exactly that length and cross-fades their latents on the device
(``sab_blend_windows``).  This module is the integer part: where the windows start and how they are grouped into
solves of bounded size.  Pure host logic, shared by ``separate()`` and the tests.
"""
from __future__ import annotations

import os
from typing import List, NamedTuple, Sequence, Tuple

# Rows (windows x candidates x window frames) of one grouped solve.  On the sam-audio-large stand-in the DiT plan takes
# about 123 KB per row (the fp32 residual stream, QKV, FFN and conditioning buffers of build_dit_plan), so 100 000 rows,
# ten windows of 10 000 frames, keep one group's plan near the codec's 12 GB chunk budget.  Measured with
# tools/longform_bench.py --only-separate on an H100 80GB HBM3 (700 W power limit): 12.32 GB of DiT plan for one group.
DEFAULT_WINDOW_ROWS = 100_000


class Window(NamedTuple):
    clip: int      # index of the clip in the batch
    start: int     # first frame of the window in the clip
    first: bool    # the clip's first window (no fade-in)
    last: bool     # the clip's last window (no fade-out)


def window_ramp(Tw: int) -> int:
    """Length of the cross-fade ramp: adjacent windows of a clip overlap by at least this many frames."""
    return Tw // 8


def clip_window_starts(n: int, Tw: int) -> List[int]:
    """Start frames of the windows of a clip of n valid frames: [0] when n <= Tw (one window [0, Tw), pad past n);
    otherwise the fewest windows whose adjacent overlaps are all >= Tw // 8, spread evenly with integer starts, the
    first at 0 and the last ending at n."""
    n, Tw = int(n), int(Tw)
    if n <= Tw:
        return [0]
    O = window_ramp(Tw)
    W = 1 + -(-(n - Tw) // (Tw - O))
    return [k * (n - Tw) // (W - 1) for k in range(W)]


def window_layout(sizes: Sequence[int], Tw: int) -> List[Window]:
    """Every window of the batch, clip by clip.  The ODE state of window w, candidate k, is sequence w * c + k."""
    out: List[Window] = []
    for b, n in enumerate(sizes):
        starts = clip_window_starts(int(n), Tw)
        out += [Window(b, s, i == 0, i == len(starts) - 1) for i, s in enumerate(starts)]
    return out


def window_rows_budget() -> int:
    """Rows of one grouped solve; SAB_WINDOW_ROWS overrides the default (tests force small groups with it)."""
    v = os.environ.get("SAB_WINDOW_ROWS")
    return int(float(v)) if v else DEFAULT_WINDOW_ROWS


def window_groups(n_windows: int, candidates: int, Tw: int, budget_rows: int) -> List[Tuple[int, int]]:
    """Consecutive [w0, w1) ranges of windows solved together: as many windows (all candidates of each) as fit the row
    budget, and at least one whatever the budget."""
    per = max(1, int(budget_rows) // (int(candidates) * int(Tw)))
    return [(w0, min(n_windows, w0 + per)) for w0 in range(0, n_windows, per)]
