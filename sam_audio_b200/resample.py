"""Index rules of the resampler (sab_resample, DESIGN.md section 3), shared by SAMAudio.resample(), streams and tests.

With g = gcd(orig, new), o = orig / g and n = new / g, output q = m * n + j (j < n) reads the K input samples
m * o + lo[j] + k, k < K; samples outside [0, L) are zero and a signal of L samples has ceil(n * L / o) outputs.  K and
lo come from the library's table (sab_resample_taps), so the filter design exists once, in C++.  The first tap
m * o + lo[j] never decreases with q, so the outputs computable from a prefix of the input are a prefix too, and the
input an output range reads is one span.  Pure integer logic apart from the one table query per rate pair.
"""
from __future__ import annotations

import math
from functools import lru_cache
from typing import Optional, Tuple

MIN_RATE, MAX_RATE = 8000, 192000


def check_rate(rate, what: str = "sample_rate") -> int:
    """A supported rate: an integer number of Hz in [8000, 192000]."""
    if isinstance(rate, bool) or int(rate) != rate or not MIN_RATE <= int(rate) <= MAX_RATE:
        raise ValueError(f"{what}={rate!r}: rates are integers in [{MIN_RATE}, {MAX_RATE}] Hz")
    return int(rate)


def rate_pair(orig: int, new: int) -> Tuple[int, int]:
    """(o, n): the pair reduced by its gcd."""
    g = math.gcd(int(orig), int(new))
    return int(orig) // g, int(new) // g


@lru_cache(maxsize=None)
def taps(orig: int, new: int) -> Tuple[int, Tuple[int, ...]]:
    """(K, lo) of the pair's table: K taps per output, lo[j] the first tap of phase j relative to m * o."""
    from . import _capi
    K, lo, _ = _capi.resample_taps(int(orig), int(new))
    return K, tuple(int(v) for v in lo)


def resampled_length(L: int, orig: int, new: int) -> int:
    """Outputs of a signal of L samples: ceil(n * L / o)."""
    o, n = rate_pair(orig, new)
    return -(-int(L) * n // o)


def first_tap(q: int, orig: int, new: int) -> int:
    o, n = rate_pair(orig, new)
    return (int(q) // n) * o + taps(orig, new)[1][int(q) % n]


def input_span(q0: int, q1: int, orig: int, new: int) -> Tuple[int, int]:
    """[i0, i1): the input indices outputs [q0, q1) read (q1 > q0), the zero fill outside the signal included."""
    K = taps(orig, new)[0]
    return first_tap(q0, orig, new), first_tap(int(q1) - 1, orig, new) + K


def outputs_ready(a: int, orig: int, new: int, length: Optional[int] = None) -> int:
    """Outputs [0, result) computable from the first `a` input samples.  While the length is unknown, an output needs
    every tap index below a (negative ones are zero); once the length is known (a == length), every output is."""
    if length is not None:
        return resampled_length(length, orig, new)
    K = taps(orig, new)[0]
    # the last tap first_tap(q) + K - 1 grows with q: find the first q whose last tap is >= a
    o, n = rate_pair(orig, new)
    lo, hi = 0, (max(0, int(a)) // o + 2) * n + n
    while lo < hi:
        mid = (lo + hi) // 2
        if first_tap(mid, orig, new) + K - 1 >= int(a):
            hi = mid
        else:
            lo = mid + 1
    return lo
