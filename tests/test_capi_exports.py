"""CPU: the C-ABI shared library loads and exports every symbol include/*.h declares; entry points
fail loudly (no fallback) when there is no GPU."""
import ctypes
import glob
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    return _capi.lib()


def declared_symbols():
    names = set()
    for h in glob.glob(os.path.join(ROOT, "include", "*.h")):
        src = re.sub(r"/\*.*?\*/", "", open(h).read(), flags=re.S)
        names |= set(re.findall(r"\b(sab_[a-z0-9_]+)\s*\(", src))
    return sorted(names)


def test_header_symbols_are_exported(lib):
    syms = declared_symbols()
    assert len(syms) >= 14
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/ but not exported"


def test_python_binding_covers_header():
    from sam_audio_b200 import _capi
    assert set(declared_symbols()) == set(_capi.EXPORTS)


def test_version_and_error_string(lib):
    assert lib.sab_version() == 1
    assert isinstance(lib.sab_last_error(), bytes)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_create_fails_loudly_without_gpu(lib):
    from sam_audio_b200 import _capi
    from sam_audio_b200.config import stand_in_config
    cfg = _capi.make_config(stand_in_config("sam-audio-tiny"))
    h = ctypes.c_void_p()
    rc = lib.sab_create(ctypes.byref(cfg), 0, ctypes.byref(h))
    assert rc != 0 and b"no CUDA device" in lib.sab_last_error()
    with pytest.raises(RuntimeError):
        from sam_audio_b200.model import build_synthetic_model
        build_synthetic_model("sam-audio-tiny")


def test_config_struct_layout_matches_header():
    """sizeof(sab_config) from the ctypes mirror == what the C side compiled (13 scalars + 5 + 2x8 ints)."""
    from sam_audio_b200 import _capi
    assert ctypes.sizeof(_capi.SabConfig) == 4 * (13 + 5 + 16)


_FAKE = 1 << 20     # a 16 B aligned non-null address: the descriptor checks run before anything is dereferenced


def _gemm_desc(**kw):
    """A valid 128 x 256 x 64 affine descriptor (fp32 output), with `kw` overriding its fields."""
    from sam_audio_b200 import _capi
    d = _capi.SabTestGemmDesc(mode=0, bn=256, bk=64, cg=1, a=_FAKE, a_cols=64, a_rows=128, a_items=1, b=_FAKE, n=256,
                              out_f32=_FAKE, out_f32_ld=256, rope_T=1)
    d.n_runs[0] = 1
    d.runs[0][0].nkb = 1
    for k, v in kw.items():
        if k == "runs":                                    # {(list, index): (row_shift, a_col, nkb)}
            for (l, i), (s, c, n) in v.items():
                d.runs[l][i].row_shift, d.runs[l][i].a_col, d.runs[l][i].nkb = s, c, n
        elif k == "n_runs":
            d.n_runs[0], d.n_runs[1] = v
        else:
            setattr(d, k, v)
    return d


def _gemm_ex_error(lib, d):
    rc = lib.sab_test_gemm_ex(ctypes.byref(d), None)
    return None if rc == 0 else lib.sab_last_error().decode()


def test_gemm_desc_struct_bytes_rejected(lib):
    """A caller compiled against another version of sab_test_gemm_desc is refused before any field is read."""
    from sam_audio_b200 import _capi
    assert ctypes.sizeof(_capi.SabTestGemmDesc) % 8 == 0
    for wrong in (ctypes.sizeof(_capi.SabTestGemmDesc) - 8, 0, 4):
        err = _gemm_ex_error(lib, _gemm_desc(struct_bytes=wrong))
        assert err is not None and "struct_bytes" in err and "header and binding differ" in err, err


_QKV = dict(mode=2, out_f32=None, out_bf16=_FAKE, out_bf16_ld=256, qnorm_w=_FAKE, knorm_w=_FAKE, n_q_end=256,
            n_k_end=256, rope_T=4)
_XA = dict(_QKV, xa_kv=_FAKE, xa_kv_ld=512, xa_v_col0=256, xa_Tk=3, xa_T=128)
_NORM_IN = dict(ssq_in=_FAKE, ssq_n=2, ssq_inv_dim=1 / 256, ibias=_FAKE, ibias_ld=256, ibias_div=128)
_B2B = dict(bn=64, bk=64, n=64, b2b=1, w1=_FAKE, b2b_bias=_FAKE, b2b_alpha=_FAKE, out_f32_ld=64)


@pytest.mark.parametrize("fields,message", [
    # the fused-norm consumer is applied only by the SwiGLU and plain QKV epilogues
    (dict(_NORM_IN), "not applied in the affine modes"),
    (dict(_NORM_IN, mode=3), "not applied in the affine modes"),
    (dict(_XA, **_NORM_IN), "not applied with fused cross-attention"),
    (dict(_QKV, ssq_in=_FAKE, ssq_n=2), "ssq_in needs ssq_n > 0 and ibias"),
    # fused cross-attention
    (dict(_XA, xa_Tk=0), "xa_Tk=0 outside 1..8"),
    (dict(_XA, xa_Tk=9), "xa_Tk=9 outside 1..8"),
    (dict(_XA, xa_T=0), "xa_T=0 must be >= 1"),
    (dict(_XA, n_q_end=128), "q-norm weights on every column"),
    (dict(xa_kv=_FAKE, xa_Tk=2, xa_T=1), "needs the QKV mode"),
    # whole heads / whole SwiGLU pairs
    (dict(_QKV, n=192), "whole 128-column heads (N=192)"),
    (dict(mode=1, n=96, out_f32=None, out_bf16=_FAKE, out_bf16_ld=48), "[32 gate | 32 up] pairs (N=96)"),
    (dict(mode=1, out_f32=None), "write out_bf16, which is not set"),
    (dict(n=100), "N=100 must be a positive multiple of 32"),
    # back-to-back residual unit
    (dict(_B2B, n=128), "back-to-back tiles need BN == N"),
    (dict(_B2B, bn=256, n=256, cg=2), "cg == 1"),
    (dict(_B2B, mode=1, out_bf16=_FAKE), "the affine mode"),
    (dict(_B2B, gate=_FAKE, gate_ld=64), "back-to-back tiles apply no gate"),
    (dict(_B2B, b2b_alpha=None), "need b2b_bias and b2b_alpha"),
    # per-item divisors
    (dict(gate=_FAKE, gate_ld=256, gate_div=0), "gate_div=0 must be > 0"),
    (dict(gate=_FAKE, gate_ld=256, gate_div=-3), "gate_div=-3 must be > 0"),
    (dict(ibias=_FAKE, ibias_div=0), "ibias_div=0 must be > 0"),
    # fused-norm producer outputs and Snake
    (dict(out_scaled=_FAKE, colscale=_FAKE), "need the AFFINE_NORM mode"),
    (dict(mode=3, out_scaled=_FAKE), "out_scaled needs colscale"),
    (dict(out_act=_FAKE, out_act_ld=256), "out_act needs snake_alpha"),
    (dict(_QKV, use_rope=1), "use_rope needs rope"),
    # schedule
    (dict(cg=2, grid_ctas=3), "grid of 3 CTAs is not a multiple of cg=2"),
    (dict(cg=3), "cg=3 must be 1 or 2"),
    (dict(reverse_m=2), "reverse_m=2 out of range"),
    # K runs
    (dict(n_period=256, n_switch=0, n_runs=(1, 2), runs={(0, 0): (0, 0, 2), (1, 0): (0, 0, 1), (1, 1): (1, 0, 2)}),
     "run lists differ in K (2 vs 3 k-blocks)"),
    (dict(n=512, n_period=384, n_switch=128, n_runs=(1, 1), runs={(1, 0): (0, 0, 1)}), "does not divide the tap switch"),
    (dict(runs={(0, 0): (0, 0, 0)}), "K run with 0 k-blocks"),
    (dict(n_runs=(9, 0)), "9 K runs (at most 8)"),
    # combinations without an instantiation
    (dict(bn=192, bk=32), "no GEMM instantiation for BN=192 BK=32 mode=0 cg=1 b2b=0"),
    (dict(bn=128, mode=2, cg=2, out_f32=None, out_bf16=_FAKE, qnorm_w=_FAKE, n_q_end=128, rope_T=1),
     "no GEMM instantiation for BN=128 BK=64 mode=2 cg=2"),
    (dict(bn=128, mode=1, out_f32=None, out_bf16=_FAKE), "no GEMM instantiation for BN=128 BK=64 mode=1 cg=1"),
    (dict(_B2B, bn=96, bk=64, n=96), "no GEMM instantiation for BN=96 BK=64 mode=0 cg=1 b2b=1"),
    (dict(mode=4), "unknown GEMM mode 4"),
])
def test_gemm_desc_rules_rejected(lib, fields, message):
    """Host-only: sab_test_gemm_ex refuses every parameter combination the kernel would silently ignore or mis-handle,
    with the rule in the message, before any CUDA call (so this runs without a GPU).  The engine's own plans pass the
    same check at every launch."""
    err = _gemm_ex_error(lib, _gemm_desc(**fields))
    assert err is not None and message in err, err


@pytest.mark.skipif(torch.cuda.is_available(), reason="the fake operands would reach the device")
def test_gemm_desc_valid_passes_the_rules(lib):
    """The base descriptor and each family's valid form pass every rule and fail only at the first CUDA call."""
    for fields in ({}, dict(_QKV), dict(_XA), dict(_QKV, **_NORM_IN), dict(_B2B), dict(cg=2, grid_ctas=4),
                   dict(mode=1, out_f32=None, out_bf16=_FAKE, **_NORM_IN), dict(mode=3, out_scaled=_FAKE, colscale=_FAKE,
                                                                              ssq_out=_FAKE, ssq_ld=2)):
        err = _gemm_ex_error(lib, _gemm_desc(**fields))
        assert err is not None and "sab_test_gemm_ex:" not in err and "struct_bytes" not in err, (fields, err)


def test_native_solver_grid_matches_the_oracle_evaluation_times(lib):
    """Host-only seam (no GPU): the evaluation times sab_solve uploads are the ones the oracle's fixed-grid solvers
    visit, in order — midpoint: exact multiples of 1/32 for 16 steps (SURVEY App. A.10); euler; rk4 (3/8 rule stages)."""
    import numpy as np
    from oracle import restate
    from sam_audio_b200 import _capi
    for name, steps in (("midpoint", 16), ("euler", 8), ("rk4", 4), ("midpoint", 5)):
        seen = []

        def f(t, y):
            seen.append(float(t))
            return -y
        restate.odeint_fixed(f, torch.ones(1), steps, name)
        n = ctypes.c_int(0)
        times = np.zeros(128, np.float32)
        _capi.check(lib.sab_test_solver_grid(_capi.Engine.ODE_METHODS[name], steps, 128, ctypes.addressof(n), times.ctypes.data))
        assert n.value == len(seen)
        assert np.allclose(times[: n.value], np.array(seen, np.float32), rtol=0, atol=1e-7), name
    n = ctypes.c_int(0)
    times = np.zeros(128, np.float32)
    _capi.check(lib.sab_test_solver_grid(0, 16, 128, ctypes.addressof(n), times.ctypes.data))
    assert times[:32].tolist() == [k / 32 for k in range(32)]            # bit-exact multiples of 1/32
    assert lib.sab_test_solver_grid(7, 4, 128, ctypes.addressof(n), times.ctypes.data) != 0 and b"unknown ODE method" in lib.sab_last_error()
