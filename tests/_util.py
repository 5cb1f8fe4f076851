import glob
import math
import os


def rel_l2(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def snr_db(a, b):
    return -20.0 * math.log10(max(rel_l2(a, b), 1e-30))


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
