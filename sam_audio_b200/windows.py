"""Windowed solving of batches longer than the model's position table (DESIGN.md section 3).

The DiT's RoPE table ends at ``transformer.max_positions`` frames (reference rope.py:152), so ``SAMAudio.separate()``
solves a longer batch as overlapping windows of exactly that length and cross-fades their latents on the device
(``sab_blend_windows``).  This module is the integer part: where the windows start and how they are grouped into
solves of bounded size, for ``separate()`` and for streams (``SAMAudio.stream()``), whose layout must not depend on
samples that have not arrived.  Pure host logic, shared by the model and the tests.
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


# ---- streams (SAMAudio.stream, DESIGN.md section 3) ----
# A stream does not know its length until flush(), so its windows cannot be spread over it: window k starts at k * H with
# H = W - O, whatever the length, and flush() adds windows until the last valid frame is covered.  Every window a stream
# has solved before flush() is therefore one of the windows of the final layout.


def stream_hop(W: int) -> int:
    """Frames between the starts of adjacent stream windows: W - window_ramp(W), so adjacent windows overlap by
    exactly window_ramp(W) frames."""
    return int(W) - window_ramp(W)


def stream_window_starts(n_final: int, W: int) -> List[int]:
    """Start frames of every window of a stream of n_final valid frames after flush(): k * H for the fewest k = 0, 1, ...
    whose windows cover [0, n_final), at least one.  The last window may run past n_final (padding, masked)."""
    n, W, H = max(1, int(n_final)), int(W), stream_hop(W)
    return [k * H for k in range(1 + max(0, -(-(n - W) // H)))]


def stream_frames_available(n_samples: int, hop: int, halo_enc: int) -> int:
    """Latent frames [0, result) the codec encoder can produce, before flush(), from the first n_samples samples: a frame
    needs halo_enc frames of samples past its own end."""
    return max(0, int(n_samples) // int(hop) - int(halo_enc))


def stream_windows_ready(n_frames: int, W: int) -> int:
    """Windows that can be solved, before flush(), once frames [0, n_frames) are encoded: those with k * H + W <= n."""
    n, W = int(n_frames), int(W)
    return 0 if n < W else (n - W) // stream_hop(W) + 1


def stream_final_frames(n_solved: int, W: int, n_final: int = -1) -> int:
    """Frames [0, result) whose latent is final once windows [0, n_solved) are solved.  Before flush() (n_final < 0) frame
    t is final when window t // H, the last window that can cover it, is solved; after flush() every window of
    stream_window_starts(n_final, W) is solved and all n_final frames are final."""
    return int(n_final) if n_final >= 0 else int(n_solved) * stream_hop(W)


def stream_emit_end(final: int, halo_dec: int, flushed: bool) -> int:
    """Frames [0, result) that can be decoded to audio: a frame needs halo_dec final frames past it, except at the end of
    the stream, where the decoder's zero fill is the clip edge."""
    return int(final) if flushed else max(0, int(final) - int(halo_dec))


def stream_window_frames(window_seconds: float, frame_rate: float, max_positions: int) -> int:
    """W = round(window_seconds * frame_rate) latent frames, checked against 8 <= W <= max_positions."""
    W = int(round(float(window_seconds) * float(frame_rate)))
    if not 8 <= W <= int(max_positions):
        raise ValueError(f"window_seconds={window_seconds} gives W={W} latent frames; a stream window needs "
                         f"8 <= W <= {int(max_positions)} (the model's position table)")
    return W


def window_rows_budget() -> int:
    """Rows of one grouped solve; SAB_WINDOW_ROWS overrides the default (tests force small groups with it)."""
    v = os.environ.get("SAB_WINDOW_ROWS")
    return int(float(v)) if v else DEFAULT_WINDOW_ROWS


def window_groups(n_windows: int, candidates: int, Tw: int, budget_rows: int) -> List[Tuple[int, int]]:
    """Consecutive [w0, w1) ranges of windows solved together: as many windows (all candidates of each) as fit the row
    budget, and at least one whatever the budget."""
    per = max(1, int(budget_rows) // (int(candidates) * int(Tw)))
    return [(w0, min(n_windows, w0 + per)) for w0 in range(0, n_windows, per)]


# ---- stream groups (SAMAudio.stream_group, DESIGN.md section 3) ----
# A tick advances several streams at once: the windows every stream makes ready are solved together, in the groups of
# window_groups, and each planned call (encode, solve, decode) runs at an item count rounded up to a bucket, so that the
# engine keeps one plan per bucket instead of planning anew whenever the number of windows in a tick changes.


def stream_group_capacity(W: int, budget_rows: int) -> int:
    """Items of the largest planned call of a stream group: the windows of one grouped solve.  A tick's encode and
    decode calls of a group never have more items than the windows solved in it (one slice per window or per stream)."""
    return max(1, int(budget_rows) // int(W))


def stream_buckets(capacity: int) -> List[int]:
    """The item counts a stream group plans calls for: the powers of two below capacity, then capacity."""
    out, b = [], 1
    while b < int(capacity):
        out.append(b)
        b *= 2
    return out + [int(capacity)]


def stream_bucket(n: int, capacity: int, resident: Sequence[int] = ()) -> List[int]:
    """Slots of a planned call of n live items: the smallest power of two >= n, capped at capacity, or, when resident
    bucket sizes are given and one of them is >= n, the smallest such (a flush reuses the plans of earlier ticks).
    Slot i < n holds item i; every spare slot repeats a live item (item i % n) and its output is dropped.  An item's
    result does not depend on the other items of its call, so the filler changes no bit."""
    n, capacity = int(n), int(capacity)
    if not 1 <= n <= capacity:
        raise ValueError(f"a planned call of {n} items in a stream group of capacity {capacity}")
    fits = [int(b) for b in resident if int(b) >= n]
    size = min(fits) if fits else next(b for b in stream_buckets(capacity) if b >= n)
    return [i % n for i in range(size)]


def stream_flush_rows(budget_rows: int, W: int, resident: Sequence[int]) -> int:
    """Row budget of the grouped solves of a flush tick: at most the largest resident bucket of windows, so that ending
    many streams at once reuses the plans of the steady ticks instead of planning a larger bucket beside them."""
    return min(int(budget_rows), max(resident) * int(W)) if resident else int(budget_rows)


# ---- offline jobs in a stream group (StreamGroup.submit, DESIGN.md section 3) ----
# A job is a stream whose whole input is known when it is submitted.  It runs only in the filler slots of a tick's
# planned calls, so its codec slices must have the lengths of the plans those calls run: the steady slices of a live
# stream (one window per tick).  Knowing its whole input, a job can cut every encode and decode into tiles of exactly
# those lengths; a kept row sees the same operands as in an un-tiled run (DESIGN.md section 3, long clips), so the tiles
# change no bit.


def stream_steady_slices(W: int, halo_enc: int, halo_dec: int) -> Tuple[int, int]:
    """Frames of a live stream's steady encode and decode slices, (H + 2 * halo_enc, H + 2 * halo_dec): the frames one
    window adds, with the codec's halo on each side."""
    H = stream_hop(W)
    return H + 2 * int(halo_enc), H + 2 * int(halo_dec)


def stream_job_min_frames(W: int, halo_enc: int, halo_dec: int) -> int:
    """Latent frames a job needs so that both its encode and its decode can be cut into tiles of the steady lengths."""
    return max(stream_steady_slices(W, halo_enc, halo_dec))


def stream_tiles(n: int, L: int, halo: int) -> List[Tuple[int, int, int]]:
    """Tiles of exactly L frames over frames [0, n): (start, keep0, keep1) per tile, the tile covering [start, start + L)
    and keeping rows [keep0, keep1).  The first tile starts at 0 and the last ends at n (right-aligned); a tile keeps
    the rows at least `halo` away from each of its cuts that is not an edge of [0, n), and the kept rows cover [0, n)
    once, in order.  Needs n >= L > 2 * halo."""
    n, L, halo = int(n), int(L), int(halo)
    if L <= 2 * halo or n < L:
        raise ValueError(f"tiles of {L} frames with a halo of {halo} over {n} frames: need n >= L > 2 * halo")
    out: List[Tuple[int, int, int]] = []
    a = 0
    while a < n:
        s = 0 if a == 0 else a - halo
        if s + L >= n:                       # the tile reaches the end: right-align it, its kept rows start at a
            out.append((n - L, a, n))
            break
        out.append((s, a, s + L - halo))
        a = s + L - halo
    return out


def stream_job_admit(offers: Sequence[int], free: int) -> List[int]:
    """Job items a planned call takes: offers[i] items are ready for the i-th job in submission order, and the call has
    `free` filler slots.  First in, first out: a job gets slots only when every earlier job has none left ready; each
    job's items are a prefix of its ready ones, so they keep their order."""
    taken, free = [], max(0, int(free))
    for n in offers:
        t = min(max(0, int(n)), free)
        taken.append(t)
        free -= t
    return taken


def stream_job_slots(n_live: int, size: int, n_jobs: int) -> List[int]:
    """Slots of a planned call of `size` slots with n_live live items and n_jobs job items: slot i < n_live + n_jobs
    holds item i (live items first), every later slot repeats a live item as stream_bucket's filler does (a job item
    when the call has none).  With n_jobs = 0 these are stream_bucket's slots."""
    n_live, size, n_jobs = int(n_live), int(size), int(n_jobs)
    n = n_live + n_jobs
    if n_live < 0 or n_jobs < 0 or not 1 <= n <= size:
        raise ValueError(f"{n_live} live and {n_jobs} job items in a call of {size} slots")
    return [i if i < n else i % (n_live or n_jobs) for i in range(size)]


def stream_drain_bucket(n: int, resident: Sequence[int]) -> int:
    """Slots of a planned call of a tick that holds only jobs (StreamGroup.drain), with n job items ready: the smallest
    resident bucket that holds them, else the largest (the rest wait for the next tick); bucket 1 when nothing is
    resident, so draining plans no bucket that the group's live ticks have not."""
    resident = [int(b) for b in resident] or [1]
    fits = [b for b in resident if b >= int(n)]
    return min(fits) if fits else max(resident)


class TickWindows(NamedTuple):
    key: object    # the stream
    ka: int        # first window of the stream solved in this group
    kb: int        # one past the last
    last: bool     # kb is the stream's k_end of this tick


def stream_tick_groups(due: Sequence[Tuple[object, int, int]], W: int, budget_rows: int) -> List[List[TickWindows]]:
    """The grouped solves of a tick.  due = [(stream, k0, k_end)], the windows [k0, k_end) each stream solves in this
    tick, in tick order.  Every window goes in order into groups of at most stream_group_capacity(W, budget_rows)
    windows (the groups of window_groups over all of them); a stream's windows inside a group are one range."""
    flat = [(key, k, k_end) for key, k0, k_end in due for k in range(int(k0), int(k_end))]
    groups: List[List[TickWindows]] = []
    for g0, g1 in window_groups(len(flat), 1, W, budget_rows):
        grp: List[TickWindows] = []
        for key, k, k_end in flat[g0:g1]:
            if grp and grp[-1].key is key:
                grp[-1] = grp[-1]._replace(kb=k + 1, last=k + 1 == k_end)
            else:
                grp.append(TickWindows(key, k, k + 1, k + 1 == k_end))
        groups.append(grp)
    return groups
