import glob
import math
import os


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def snr_db(a, b):
    return -20.0 * math.log10(max(rel_l2(a, b), 1e-30))


def snake_bound(v, a):
    """|__sinf / rcp.approx Snake - exact| for input v, alpha a: sin.approx.f32 has an absolute error of 2^-21.41 on
    [-pi, pi], and the fp32 range reduction outside it about one ulp of the scaled argument, 2^-22 |a v|; d/dv sin^2(a v) / a
    is bounded by 2, so the activation's error is 2 (2^-21.41 + 2^-22 |a v|) / a, plus 2^-21 / a for the reciprocal."""
    d_sin = 2.0 ** -21.41 + 2.0 ** -22 * (a * v).abs()
    return (2 * d_sin + 2.0 ** -21) / a


def _merge(a, b):
    for k, v in b.items():
        if isinstance(v, dict) and isinstance(a.get(k), dict):
            _merge(a[k], v)
        else:
            a[k] = v
    return a


def load_golden(golden_dir, name):
    """A fixture stored as <name>.pt plus optional parts <name>.1.pt, <name>.2.pt, ... (each file stays under 1 MB)
    whose nested dicts merge into one."""
    import torch
    g = torch.load(os.path.join(golden_dir, name + ".pt"))
    for part in sorted(glob.glob(os.path.join(golden_dir, glob.escape(name) + ".[0-9]*.pt"))):
        _merge(g, torch.load(part))
    return g
