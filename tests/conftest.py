import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def usable_host_cores() -> int:
    """Cores this process may actually use: the smaller of the affinity mask and the cgroup CPU quota.  GPU boxes
    report 128 logical CPUs under a 16-core quota; torch's default (one thread per logical CPU) then oversubscribes
    and the CPU oracle legs of the parity tests run several times slower, more so on a busy host."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    for quota_file, period_file in (("/sys/fs/cgroup/cpu.max", None),
                                    ("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "/sys/fs/cgroup/cpu/cpu.cfs_period_us")):
        try:
            if period_file is None:
                q, per = open(quota_file).read().split()
            else:
                q, per = open(quota_file).read().strip(), open(period_file).read().strip()
            if q not in ("max", "-1"):
                n = max(1, min(n, int(float(q) / float(per) + 0.5)))
            break
        except Exception:
            continue
    return n


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (select with -m gpu)")
    import torch
    torch.set_num_threads(usable_host_cores())


@pytest.fixture(scope="session")
def golden_dir():
    return GOLDEN


@pytest.fixture(scope="session")
def tiny_cfg():
    from sam_audio_b200.config import stand_in_config
    return stand_in_config("sam-audio-tiny")


@pytest.fixture(scope="session")
def tiny_sd(tiny_cfg):
    from sam_audio_b200.synthetic import make_state_dict
    return make_state_dict(tiny_cfg, seed=0)


@pytest.fixture(scope="session")
def tiny_model(tiny_cfg):
    """Session-wide tiny model on cuda:0 (gpu tests only)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.model import build_synthetic_model
    return build_synthetic_model("sam-audio-tiny", seed=0, device="cuda:0")
