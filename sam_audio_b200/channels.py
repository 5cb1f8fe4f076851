"""Index rules of the multichannel stems (sab_spread_channels, DESIGN.md section 3), shared by
SAMAudio.spread_channels(), streams and tests.

At the codec's rate, frame j >= 0 covers samples [j a - 3 a, j a + a) with N = 2048 and hop a = 512, so sample s >= 0
lies in the frames floor(s / a) .. floor(s / a) + 3.  A frame is computable once the mono target and residual and the
channels are known through its end (or their lengths are known), and a sample is emitted once its last frame is
computable.  So the samples a stream can emit from prefixes of its inputs are a prefix too, whole hops of a until the
lengths are known, and a sample waits at most 4 a = 2048 samples (42.7 ms at 48 kHz) for inputs past it.  Pure integer
logic.
"""
from __future__ import annotations

from typing import Optional, Tuple

N = 2048                  # frame length
HOP = 512                 # hop a = N / 4
LATENCY = 4 * HOP         # a sample is emitted once every input is known 4 a past its hop's start


def frames_of(s: int) -> Tuple[int, int]:
    """[j0, j1): the frames covering sample s >= 0."""
    return int(s) // HOP, int(s) // HOP + 4


def frame_span(j: int) -> Tuple[int, int]:
    """[i0, i1): the samples frame j covers (negative ones read as zero)."""
    return int(j) * HOP - 3 * HOP, int(j) * HOP + HOP


def input_span(s0: int, s1: int) -> Tuple[int, int]:
    """[i0, i1): the input indices outputs [s0, s1) read (s1 > s0), the zero fill outside the signals included."""
    return frame_span(int(s0) // HOP)[0], frame_span((int(s1) - 1) // HOP + 3)[1]


def keep_from(produced: int) -> int:
    """The first input sample a later output (from `produced` on) reads: inputs before it can be dropped."""
    return max(0, input_span(produced, produced + 1)[0])


def spread_ready(tr_received: int, x_received: int, tr_length: Optional[int] = None,
                 x_length: Optional[int] = None) -> int:
    """Outputs [0, result) computable when the mono stems are known on [0, tr_received) and the channels on [0,
    x_received); an input whose length is known (not None) is known everywhere, its zero fill included.  Once the stems'
    length is known, every output up to it can be ready; the outputs never pass it."""
    known = [r for r, L in ((tr_received, tr_length), (x_received, x_length)) if L is None]
    if not known:
        return int(tr_length)
    # sample s needs frame floor(s / a) + 3, which ends at (floor(s / a) + 4) a
    ready = max(0, (min(known) // HOP - 3) * HOP)
    return ready if tr_length is None else min(ready, int(tr_length))


def check_spread_shapes(target, residual, mixture) -> Tuple[int, int, int]:
    """(C, S, S') of SAMAudio.spread_channels' arguments: target and residual [S'], mixture [C, S] with 1 <= C <= 8 and
    1 <= S <= S'.  Raises ValueError otherwise."""
    import torch
    from .stream import MAX_CHANNELS
    for name, t in (("target", target), ("residual", residual), ("mixture", mixture)):
        if not isinstance(t, torch.Tensor):
            raise ValueError(f"spread_channels() takes tensors, got {type(t).__name__} for {name}")
    if target.dim() != 1 or residual.shape != target.shape or target.shape[0] < 1:
        raise ValueError(f"spread_channels() takes a mono target and residual of one length [S'], got "
                         f"{tuple(target.shape)} and {tuple(residual.shape)}")
    if mixture.dim() != 2 or not 1 <= mixture.shape[0] <= MAX_CHANNELS or not 1 <= mixture.shape[1] <= target.shape[0]:
        raise ValueError(f"spread_channels() takes a mixture [C, S] with 1 <= C <= {MAX_CHANNELS} and 1 <= S <= S' = "
                         f"{target.shape[0]} (the stems' length), got {tuple(mixture.shape)}")
    return mixture.shape[0], mixture.shape[1], target.shape[0]
