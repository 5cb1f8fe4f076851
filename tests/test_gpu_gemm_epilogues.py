"""GPU (H100): every fused epilogue of the wgmma GEMM (sam_audio_b200/csrc/gemm_tc.cuh), the conv K-run lists and the
persistent tile schedule, through sab_test_gemm_ex (the engine's own planner and instantiation table), element by
element against a float64 reference computed from the bf16 operands the kernel reads.

Bounds, per element, with rms_row = the RMS of the reference row:
  * fp32 outputs ..................................... |o - r| <= 1e-3 rms_row
  * bf16 outputs ..................................... |o - r| <= 2^-8 |r| + 1e-3 rms_row   (round to nearest: 2^-8)
  * Snake (__sinf, rcp.approx): sin.approx.f32 has an absolute error of 2^-21.41 on [-pi, pi]; outside it the fp32
    range reduction adds about one ulp of the scaled argument, 2^-22 |a v|.  d/dv sin^2(a v) / a is bounded by 2, so the
    activation's error is 2 (2^-21.41 + 2^-22 |a v|) / a, plus 2^-21 / a for rcp.approx, plus 2x the fp32 error of v.
  * back-to-back: the intermediate Snake tile is rounded to bf16 inside the kernel.  Where its exact value lies within
    the Snake bound of a bf16 rounding midpoint, kernel and reference may round it to neighbouring values: such
    elements get one bf16 ulp of slack, the others the Snake bound; both are carried through |W1| into the output.
  * fused cross-attention (ex2.approx: relative error 2^-22; IEEE 1/den): the probability error is ~1e-6 relative, far
    below the 1e-3 rms_row term, so the bf16 bound applies unchanged.
  * schedule variants (grid size, group_m, serpentine order, 1- vs 2-CTA tiles): bit-identical, no tolerance.
Every output has guard columns (ld > N) and guard rows filled with a sentinel that must survive.
"""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

from _util import rel_l2, snake_bound

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AFFINE, SWIGLU, QKV, AFFINE_NORM = 0, 1, 2, 3
SENT = -7776.0            # exactly representable in bf16 and fp32
DEV = "cuda"
LOG2E = 1.4426950408889634


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    assert torch.cuda.is_available()
    return _capi


# ------------------------------------------------------------------------------------------------ helpers
class Out:
    """An output matrix [rows, cols] inside a sentinel-filled buffer with 8 guard columns and 3 guard rows."""

    def __init__(self, rows, cols, dtype):
        self.rows, self.cols, self.ld = rows, cols, cols + 8
        self.buf = torch.full((rows + 3, self.ld), SENT, dtype=dtype, device=DEV)

    def reset(self):
        self.buf.fill_(SENT)

    @property
    def val(self):
        return self.buf[: self.rows, : self.cols]

    def assert_guards(self, what):
        keep = torch.ones_like(self.buf, dtype=torch.bool)
        keep[: self.rows, : self.cols] = False
        bad = int((self.buf[keep].float() != SENT).sum())
        assert bad == 0, f"{what}: {bad} writes outside the [{self.rows}, {self.cols}] output"
        assert torch.isfinite(self.val.float()).all(), f"{what}: non-finite or unwritten outputs"


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(g, *shape, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=g) * scale


def bf(x):
    return x.bfloat16()


def row_rms(r):
    return r.pow(2).mean(-1, keepdim=True).sqrt()


def assert_close(o, r, what, bf16=False, extra=0.0, rms=None):
    """Element-wise bound (module docstring); `extra` adds a per-element term, `rms` overrides the row RMS."""
    r = r.double()
    rms = row_rms(r) if rms is None else rms
    tol = 1e-3 * rms + extra + (2.0 ** -8 * r.abs() if bf16 else 0.0)
    err = (o.double() - r).abs()
    bad = err > tol
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound; first at flat index {i}: "
                             f"got {float(o.flatten()[i])}, want {float(r.flatten()[i])}, bound {float(tol.flatten()[i])}; "
                             f"max err/bound {float((err / tol).max()):.3g}")


def snake(v, a):
    return v + torch.sin(a * v) ** 2 / (a + 1e-9)


def bf16_mismatch_bound(m, delta):
    """Bound on |bf16(m') - bf16(m)| for |m' - m| <= delta: delta, plus one ulp where m lies within delta of a
    rounding midpoint (the two may round to neighbours)."""
    _, e = torch.frexp(m)
    ulp = torch.ldexp(torch.ones_like(m), (e - 8).to(torch.int32))
    to_mid = ulp / 2 - (m - m.bfloat16().double()).abs()
    return delta + torch.where(to_mid <= delta, ulp, torch.zeros_like(m))


def launch(capi, runs, **fields):
    d = capi.SabTestGemmDesc()
    names = {f[0] for f in d._fields_}
    for l, rl in enumerate(runs):
        d.n_runs[l] = len(rl)
        for i, (s, c, n) in enumerate(rl):
            d.runs[l][i].row_shift, d.runs[l][i].a_col, d.runs[l][i].nkb = s, c, n
    for k, v in fields.items():
        assert k in names, k
        if isinstance(v, Out):
            setattr(d, k, v.buf.data_ptr())
            setattr(d, "ssq_ld" if k == "ssq_out" else k + "_ld", v.ld)
        elif torch.is_tensor(v):
            setattr(d, k, v.data_ptr())
        else:
            setattr(d, k, v)
    capi.check(capi.lib().sab_test_gemm_ex(ctypes.byref(d), capi.stream_ptr()))
    torch.cuda.synchronize()


def ref_acc(A3, B, runs, bk, bn=256, n_period=0, n_switch=0):
    """sum over the K runs of the row-shifted, column-offset A block x its B slice (rows outside an item read as zero,
    columns past the view's width too).  A3: [items, T, cols] (the visible view); returns fp64 [items * T, N]."""
    A3, B = A3.double(), B.double()
    items, T, cols = A3.shape
    outs = []
    for rl in runs:
        acc = torch.zeros(items, T, B.shape[0], dtype=torch.float64, device=DEV)
        k0 = 0
        for s, c, nkb in rl:
            w = nkb * bk
            blk = torch.zeros(items, T, w, dtype=torch.float64, device=DEV)
            lo, hi, c1 = max(0, -s), min(T, T - s), min(cols, c + w)
            if hi > lo and c1 > c:
                blk[:, lo:hi, : c1 - c] = A3[:, lo + s: hi + s, c:c1]
            acc += blk @ B[:, k0: k0 + w].t()
            k0 += w
        outs.append(acc.reshape(items * T, -1))
    if n_period == 0:
        return outs[0]
    n0 = torch.arange(B.shape[0], device=DEV) // bn * bn
    return torch.where((n0 % n_period) >= n_switch, outs[1], outs[0])


def linear_runs(K, bk):
    return [[(0, 0, K // bk)]]


# ------------------------------------------------------------------------------------------------ cases
class Case:
    """One launch: descriptor fields, its outputs, and the reference check.  `run` refills the outputs first."""

    def __init__(self, capi, runs, fields, outs, check):
        self.capi, self.runs, self.fields, self.outs, self.check = capi, runs, fields, outs, check

    def run(self, **override):
        for o in self.outs.values():
            o.reset()
        launch(self.capi, self.runs, **dict(self.fields, **override))
        for k, o in self.outs.items():
            o.assert_guards(k)
        return {k: o.val.clone() for k, o in self.outs.items()}


def affine_case(capi, bn, bk, cg, T=300, items=2, N=None, K=None, relu=0, bias_mod=0, gate_div=77, seed=0,
                outputs=("out_f32", "out_bf16", "out_act"), lda_pad=64):
    """(acc + bias[n % bias_mod]) * gate[row / gate_div, n] * alpha + res -> relu -> fp32 | bf16 | Snake bf16, A a column
    slice of a wider buffer (row pitch > K)."""
    g = gen(seed)
    N = N or bn + 32                      # last n-tile: one 32-column chunk
    K = K or 3 * 64
    M = T * items
    A_full = bf(randn(g, M, K + lda_pad))
    B = bf(randn(g, N, K, scale=K ** -0.5))
    bias = randn(g, bias_mod or N, scale=0.5)
    n_gate = (M - 1) // gate_div + 1
    gate = 1 + 0.25 * randn(g, n_gate, N + 4)
    res = randn(g, M, N)
    res_buf = torch.zeros(M, N + 4, device=DEV)
    res_buf[:, :N] = res
    sal = 0.5 + torch.rand(bias_mod or N, device=DEV, generator=g)
    outs = {"out_f32": Out(M, N, torch.float32), "out_bf16": Out(M, N, torch.bfloat16),
            "out_act": Out(M, N, torch.bfloat16)}
    outs = {k: v for k, v in outs.items() if k in outputs}
    fields = dict(mode=AFFINE, bn=bn, bk=bk, cg=cg, a=A_full, a_cols=K, a_rows=M, a_items=1, a_row_pitch=K + lda_pad,
                  b=B, n=N, bias=bias, bias_mod=bias_mod, gate=gate, gate_ld=N + 4, gate_div=gate_div, alpha=0.75,
                  relu=relu, res=res_buf, res_ld=N + 4, snake_alpha=sal, **outs)
    runs = linear_runs(K, bk)

    def check(got):
        n = torch.arange(N, device=DEV)
        acc = ref_acc(A_full[:, :K].view(1, M, K), B, runs, bk)
        v = acc + bias.double()[n % bias_mod if bias_mod else n]
        v = v * gate.double()[torch.arange(M, device=DEV) // gate_div][:, :N] * 0.75 + res.double()
        if relu:
            v = v.clamp_min(0)
        rms = row_rms(v)
        if "out_f32" in got:
            assert_close(got["out_f32"], v, "out_f32")
        if "out_bf16" in got:
            assert_close(got["out_bf16"], v, "out_bf16", bf16=True)
        if "out_act" in got:
            a = sal.double()[n % bias_mod if bias_mod else n]
            assert_close(got["out_act"], snake(v, a), "out_act (Snake)", bf16=True, rms=2 * rms,
                         extra=snake_bound(v, a))
    return Case(capi, runs, fields, outs, check)


AFFINE_TILES = [(256, 64, 1), (256, 64, 2), (192, 64, 1), (128, 64, 1), (96, 64, 1), (64, 64, 1), (96, 32, 1),
                (128, 32, 1)]


@pytest.mark.parametrize("relu,bias_mod", [(0, 0), (1, 160)])
@pytest.mark.parametrize("bn,bk,cg", AFFINE_TILES)
def test_affine_epilogue(capi, bn, bk, cg, relu, bias_mod):
    """Every affine instantiation with the whole epilogue at once: bias (bias_mod), gate rows changing inside a tile
    (gate_div = 77), alpha, fp32 residual, relu, and fp32 + bf16 + Snake outputs; partial last n-tile."""
    c = affine_case(capi, bn, bk, cg, relu=relu, bias_mod=bias_mod, seed=bn + bk + cg + relu)
    c.check(c.run())


@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("T", [1, 77, 129, 250, 300])
def test_ragged_rows_per_item(capi, T, cg):
    """Tiles never straddle items: rows_per_item 1 .. 300 over 3 items (for cg = 2 and T <= 128 the second CTA of the
    cluster has no valid rows); N = BN + 32."""
    g = gen(T + cg)
    items, K, N = 3, 128, 288
    A = bf(randn(g, items, T, K))
    B = bf(randn(g, N, K, scale=K ** -0.5))
    bias = randn(g, N)
    out = Out(items * T, N, torch.float32)
    runs = linear_runs(K, 64)
    launch(capi, runs, mode=AFFINE, bn=256, bk=64, cg=cg, a=A, a_cols=K, a_rows=T, a_items=items, b=B, n=N, bias=bias,
           out_f32=out)
    out.assert_guards("out_f32")
    assert_close(out.val, ref_acc(A, B, runs, 64) + bias.double(), "out_f32")


def conv_case(capi, kind, seed=0):
    g = gen(seed)
    items = 2
    if kind.startswith("dil"):                         # Conv1d(C, C, k=7, dilation) 'same' (codec residual unit)
        dil, T, C = int(kind[3:]), 250, 128
        runs = [[((k - 3) * dil, 0, C // 64) for k in range(7)]]
        A = bf(randn(g, items, T, C))
        view = dict(a=A, a_cols=C, a_rows=T, a_items=items)
        A3, N, bn, extra = A, C, 128, {}
    elif kind == "down":                               # strided Conv1d(C, 2C, k=2s, stride s): taps -1 / 0 / +1
        s, C, To = 4, 64, 100
        pd = s // 2
        runs = [[(-1, (s - pd) * C, pd * C // 64), (0, 0, s * C // 64), (1, 0, (s - pd) * C // 64)]]
        A = bf(randn(g, items, To, s * C))
        view = dict(a=A, a_cols=s * C, a_rows=To, a_items=items)
        A3, N, bn, extra = A, 2 * C, 128, {}
    else:                                              # ConvTranspose1d(C, Co, k=2s, stride s): two run lists
        s, C, Co, T = 4, 128, 64, 120
        runs = [[(0, 0, C // 64), (-1, 0, C // 64)], [(0, 0, C // 64), (1, 0, C // 64)]]
        A = bf(randn(g, items, T, C))
        view = dict(a=A, a_cols=C, a_rows=T, a_items=items)
        A3, N, bn = A, s * Co, 128
        extra = dict(n_period=s * Co, n_switch=(s // 2) * Co, bias_mod=Co)
    K = sum(n for _, _, n in runs[0]) * 64
    B = bf(randn(g, N, K, scale=K ** -0.5))
    bias = randn(g, extra.get("bias_mod") or N)
    out = Out(A3.shape[0] * A3.shape[1], N, torch.float32)
    fields = dict(mode=AFFINE, bn=bn, bk=64, cg=1, b=B, n=N, bias=bias, out_f32=out, **view, **extra)

    def check(got):
        acc = ref_acc(A3, B, runs, 64, bn, extra.get("n_period", 0), extra.get("n_switch", 0))
        n = torch.arange(N, device=DEV)
        bm = extra.get("bias_mod", 0)
        assert_close(got["out_f32"], acc + bias.double()[n % bm if bm else n], f"conv {kind}")
    return Case(capi, runs, fields, {"out_f32": out}, check)


@pytest.mark.parametrize("kind", ["dil1", "dil3", "dil9", "down", "transpose"])
def test_conv_k_runs(capi, kind):
    """The conv lowering: k = 7 dilated taps (row_shift, zero rows at item edges), the encoder's strided down-sampling
    runs (-1 / 0 / +1 with an a_col offset), and the decoder's two-list ConvTranspose layout with bias_mod = Co."""
    c = conv_case(capi, kind)
    c.check(c.run())


def b2b_case(capi, bn, bk, seed=0):
    """Codec residual unit in one launch: Snake(conv7(x) + b0) -> bf16 -> @ W1^T + bias + res -> fp32 and Snake bf16."""
    g = gen(seed)
    items, T, C = 3, 250, bn
    runs = [[((k - 3) * 3, 0, C // bk) for k in range(7)]]
    A = bf(randn(g, items, T, C))
    K = 7 * C
    B = bf(randn(g, C, K, scale=K ** -0.5))
    W1 = bf(randn(g, C, C, scale=C ** -0.5))
    b0, bias = randn(g, C, scale=0.5), randn(g, C, scale=0.5)
    a0, a1 = 0.5 + torch.rand(C, device=DEV, generator=g), 0.5 + torch.rand(C, device=DEV, generator=g)
    M = items * T
    res = randn(g, M, C)
    outs = {"out_f32": Out(M, C, torch.float32), "out_act": Out(M, C, torch.bfloat16)}
    fields = dict(mode=AFFINE, bn=bn, bk=bk, cg=1, b2b=1, a=A, a_cols=C, a_rows=T, a_items=items, b=B, n=C, w1=W1,
                  b2b_bias=b0, b2b_alpha=a0, bias=bias, res=res, res_ld=C, snake_alpha=a1, **outs)

    def check(got):
        x = ref_acc(A, B, runs, bk) + b0.double()
        m = snake(x, a0.double())
        # kernel's pre-rounding intermediate: Snake bound + twice the fp32 error of x (bounded by 1e-5 of its row RMS)
        dm = bf16_mismatch_bound(m, snake_bound(x, a0.double()) + 2e-5 * row_rms(x))
        v = m.bfloat16().double() @ W1.double().t() + bias.double() + res.double()
        slack = dm @ W1.double().abs().t()
        assert_close(got["out_f32"], v, "b2b out_f32", extra=slack)
        assert_close(got["out_act"], snake(v, a1.double()), "b2b out_act", bf16=True, rms=2 * row_rms(v),
                     extra=2 * slack + snake_bound(v, a1.double()))
    return Case(capi, runs, fields, outs, check)


@pytest.mark.parametrize("bn,bk", [(64, 64), (96, 32), (128, 64)])
def test_b2b_residual_unit(capi, bn, bk):
    c = b2b_case(capi, bn, bk, seed=bn)
    c.check(c.run())


def norm_inputs(g, M, N, rows_per_item, K):
    """Fused-norm consumer inputs: positive partial sums of squares [M, 4] and a per-item bias row [items, N]."""
    ssq = torch.rand(M, 4, device=DEV, generator=g) * 0.5 * K + 0.1
    ibias = randn(g, (M - 1) // rows_per_item + 1, N + 4, scale=0.3)
    return ssq, ibias


def apply_norm_in(acc, ssq, ibias, div, K, eps):
    M, N = acc.shape
    rstd = (ssq.double().sum(1, keepdim=True) / K + eps).rsqrt()
    return rstd * acc + ibias.double()[torch.arange(M, device=DEV) // div][:, :N]


def swiglu_case(capi, cg, norm, seed=0, T=250, items=5):
    g = gen(seed)
    K, N = 256, 2 * 256 + 64                 # last n-tile: one [32 gate | 32 up] pair
    M = T * items
    A = bf(randn(g, M, K))
    B = bf(randn(g, N, K, scale=K ** -0.5))
    ssq, ibias = norm_inputs(g, M, N, T, K)
    out = Out(M, N // 2, torch.bfloat16)
    fields = dict(mode=SWIGLU, bn=256, bk=64, cg=cg, a=A, a_cols=K, a_rows=M, a_items=1, b=B, n=N, out_bf16=out, eps=1e-5)
    if norm:
        fields.update(ssq_in=ssq, ssq_n=4, ssq_inv_dim=1.0 / K, ibias=ibias, ibias_ld=N + 4, ibias_div=T)
    runs = linear_runs(K, 64)

    def check(got):
        x = ref_acc(A.view(1, M, K), B, runs, 64)
        if norm:
            x = apply_norm_in(x, ssq, ibias, T, K, 1e-5)
        x = x.view(M, N // 64, 2, 32)
        y = (torch.nn.functional.silu(x[:, :, 0]) * x[:, :, 1]).reshape(M, N // 2)
        assert_close(got["out_bf16"], y, "swiglu", bf16=True)
    return Case(capi, runs, fields, {"out_bf16": out}, check)


@pytest.mark.parametrize("norm", [0, 1])
@pytest.mark.parametrize("cg", [1, 2])
def test_swiglu(capi, cg, norm):
    c = swiglu_case(capi, cg, norm, seed=cg + 2 * norm)
    c.check(c.run())


def rope_table(n_pos, g):
    ang = torch.rand(n_pos, 64, device=DEV, generator=g, dtype=torch.float64) * 2 * math.pi
    return torch.stack([ang.cos(), ang.sin()], -1).float().contiguous()       # [n_pos, 64] (cos, sin) pairs


def qkv_ref(x, w_q, w_k, n_q_end, n_k_end, rope, pos, eps, period=0, w_stride=0):
    """Per 128-column head: RMSNorm (q columns [0, n_q_end), k columns [n_q_end, n_k_end), modulo `period`) with the
    repeat's weights, then RoPE on adjacent pairs; the other columns pass through."""
    M, N = x.shape
    y = x.clone()
    for h0 in range(0, N, 128):
        rep, hp = (h0 // period, h0 % period) if period else (0, h0)
        if hp < n_q_end:
            w = w_q[rep * w_stride: rep * w_stride + 128]
        elif hp < n_k_end:
            w = w_k[rep * w_stride: rep * w_stride + 128]
        else:
            continue
        v = x[:, h0: h0 + 128]
        v = v * (v.pow(2).mean(1, keepdim=True) + eps).rsqrt() * w.double()
        if rope is not None:
            cs = rope.double()[pos]                                            # [M, 64, 2]
            a, b = v[:, 0::2], v[:, 1::2]
            v = torch.stack([a * cs[..., 0] - b * cs[..., 1], a * cs[..., 1] + b * cs[..., 0]], -1).reshape(M, 128)
        y[:, h0: h0 + 128] = v
    return y


def qkv_case(capi, bn, cg, use_rope, norm, seed=0, T=250, items=3):
    g = gen(seed)
    d, K = 256, 256
    N = 2 * d + 128                          # q | k | v, V narrower than a tile: partial last n-tile at BN = 256
    M = T * items
    A = bf(randn(g, M, K))
    B = bf(randn(g, N, K, scale=K ** -0.5))
    wq, wk = 1 + 0.3 * randn(g, 128), 1 + 0.3 * randn(g, 128)
    rope = rope_table(T, g)
    ssq, ibias = norm_inputs(g, M, N, T, K)
    out = Out(M, N, torch.bfloat16)
    fields = dict(mode=QKV, bn=bn, bk=64, cg=cg, a=A, a_cols=K, a_rows=M, a_items=1, b=B, n=N, out_bf16=out,
                  qnorm_w=wq, knorm_w=wk, n_q_end=d, n_k_end=2 * d, rope=rope, rope_T=T, use_rope=use_rope, eps=1e-5)
    if norm:
        fields.update(ssq_in=ssq, ssq_n=4, ssq_inv_dim=1.0 / K, ibias=ibias, ibias_ld=N + 4, ibias_div=T)
    runs = linear_runs(K, 64)

    def check(got):
        x = ref_acc(A.view(1, M, K), B, runs, 64)
        if norm:
            x = apply_norm_in(x, ssq, ibias, T, K, 1e-5)
        pos = torch.arange(M, device=DEV) % T
        y = qkv_ref(x, wq, wk, d, 2 * d, rope if use_rope else None, pos, 1e-5)
        assert_close(got["out_bf16"], y, "qkv", bf16=True)
    return Case(capi, runs, fields, {"out_bf16": out}, check)


@pytest.mark.parametrize("norm", [0, 1])
@pytest.mark.parametrize("use_rope", [0, 1])
@pytest.mark.parametrize("bn,cg", [(128, 1), (256, 1), (256, 2)])
def test_qkv(capi, bn, cg, use_rope, norm):
    """q-norm / k-norm / pass-through V column ranges, RoPE at position row % rope_T over several items, and the
    fused-norm consumer (rstd * acc + ibias, V columns included)."""
    c = qkv_case(capi, bn, cg, use_rope, norm, seed=bn + cg + 2 * use_rope + 4 * norm)
    c.check(c.run())


def test_qkv_all_layers_kv_layout(capi):
    """The all-layers cross K|V GEMM: per repeat of qkv_period = 2d columns, k-norm on the first d (with that layer's
    norm weights, norm_w_stride = 128 apart) and V passed through."""
    g = gen(7)
    d, K, NL, L, items = 256, 256, 3, 5, 4
    N, M = 2 * d * NL, L * items
    A = bf(randn(g, M, K))
    B = bf(randn(g, N, K, scale=K ** -0.5))
    w_all = 1 + 0.3 * randn(g, 128 * NL)
    out = Out(M, N, torch.bfloat16)
    runs = linear_runs(K, 64)
    launch(capi, runs, mode=QKV, bn=256, bk=64, cg=1, a=A, a_cols=K, a_rows=M, a_items=1, b=B, n=N, out_bf16=out,
           qnorm_w=w_all, knorm_w=w_all, n_q_end=0, n_k_end=d, qkv_period=2 * d, norm_w_stride=128, rope_T=L, eps=1e-5)
    out.assert_guards("out_bf16")
    y = qkv_ref(ref_acc(A.view(1, M, K), B, runs, 64), w_all, w_all, 0, d, None, None, 1e-5, period=2 * d, w_stride=128)
    assert_close(out.val, y, "kv all layers", bf16=True)


def xattn_case(capi, Tk, cand, cg=1, seed=0):
    """cross.wq with the attention to the clip's text tokens fused into its epilogue: K|V read from layer 1 of a
    3-layer buffer (xa_kv_ld = 6d > 2d, xa_v_col0 = d), ragged text mask, candidates sharing their clip's K/V."""
    g = gen(seed)
    d, K, T, B_clips, NL = 256, 256, 100, 2, 3
    M = B_clips * cand * T
    A = bf(randn(g, M, K))
    W = bf(randn(g, d, K, scale=K ** -0.5))
    wq = 1 + 0.3 * randn(g, 128)
    kv_ld = 2 * d * NL
    kv = bf(randn(g, B_clips * Tk, kv_ld))
    kv_l = kv[:, 2 * d: 4 * d]                         # layer 1's K | V
    mask = torch.ones(B_clips, Tk, dtype=torch.uint8, device=DEV)
    mask[1, max(1, Tk - 2):] = 0
    out = Out(M, d, torch.bfloat16)
    fields = dict(mode=QKV, bn=256, bk=64, cg=cg, a=A, a_cols=K, a_rows=M, a_items=1, b=W, n=d, out_bf16=out,
                  qnorm_w=wq, knorm_w=wq, n_q_end=d, n_k_end=d, rope_T=T, eps=1e-5,
                  xa_kv=kv.data_ptr() + 2 * d * 2, xa_kv_ld=kv_ld, xa_v_col0=d, xa_Tk=Tk, xa_T=T * cand, xa_mask=mask,
                  xa_scale_log2=LOG2E / math.sqrt(128))
    runs = linear_runs(K, 64)

    def check(got):
        q = qkv_ref(ref_acc(A.view(1, M, K), W, runs, 64), wq, wq, d, d, None, None, 1e-5)
        clip = torch.arange(M, device=DEV) // (T * cand)
        Kt = kv_l[:, :d].double().contiguous().view(B_clips, Tk, d // 128, 128)[clip]      # [M, Tk, H, 128]
        Vt = kv_l[:, d:].double().contiguous().view(B_clips, Tk, d // 128, 128)[clip]
        s = torch.einsum("mhc,mjhc->mhj", q.view(M, d // 128, 128), Kt) / math.sqrt(128)
        s = s.masked_fill(~mask.bool()[clip][:, None, :], float("-inf"))
        o = torch.einsum("mhj,mjhc->mhc", torch.softmax(s, -1), Vt).reshape(M, d)
        assert_close(got["out_bf16"], o, "fused cross-attention", bf16=True)
    return Case(capi, runs, fields, {"out_bf16": out}, check)


@pytest.mark.parametrize("cand", [1, 3])
@pytest.mark.parametrize("Tk", [1, 3, 8])
def test_fused_cross_attention(capi, Tk, cand):
    c = xattn_case(capi, Tk, cand, seed=Tk + 10 * cand)
    c.check(c.run())


def norm_producer_case(capi, cg, seed=0, T=250, items=5):
    """EPI_AFFINE_NORM: v = (acc + bias) * gate + res -> out_f32, out_scaled = bf16(v * colscale[row / gate_div]) and
    ssq_out[row, 2 nt + parity] = sum of v^2 over the n-tile's even / odd 32-column chunks."""
    g = gen(seed)
    K, N = 256, 3 * 256 + 64                 # four n-tiles, the last one two chunks wide
    M = T * items
    n_tiles = (N + 255) // 256
    A = bf(randn(g, M, K))
    B = bf(randn(g, N, K, scale=K ** -0.5))
    bias = randn(g, N, scale=0.5)
    gate = 1 + 0.25 * randn(g, items, N)
    colscale = 1 + 0.25 * randn(g, items, N)
    res = randn(g, M, N)
    outs = {"out_f32": Out(M, N, torch.float32), "out_scaled": Out(M, N, torch.bfloat16),
            "ssq_out": Out(M, 2 * n_tiles, torch.float32)}
    fields = dict(mode=AFFINE_NORM, bn=256, bk=64, cg=cg, a=A, a_cols=K, a_rows=M, a_items=1, b=B, n=N, bias=bias,
                  gate=gate, gate_ld=N, gate_div=T, res=res, res_ld=N, colscale=colscale, colscale_ld=N, **outs)
    runs = linear_runs(K, 64)

    def check(got):
        item = torch.arange(M, device=DEV) // T
        v = (ref_acc(A.view(1, M, K), B, runs, 64) + bias.double()) * gate.double()[item] + res.double()
        assert_close(got["out_f32"], v, "norm producer out_f32")
        assert_close(got["out_scaled"], v * colscale.double()[item], "out_scaled", bf16=True)
        sq = torch.zeros(M, 2 * n_tiles, dtype=torch.float64, device=DEV)
        for c0 in range(0, N, 32):
            sq[:, 2 * (c0 // 256) + (c0 // 32) % 2] += v[:, c0: c0 + 32].pow(2).sum(1)
        assert_close(got["ssq_out"], sq, "ssq_out")
    return Case(capi, runs, fields, outs, check)


@pytest.mark.parametrize("cg", [1, 2])
def test_fused_norm_producer(capi, cg):
    c = norm_producer_case(capi, cg, seed=cg)
    c.check(c.run())


@pytest.mark.parametrize("consumer", ["swiglu", "qkv"])
def test_fused_norm_chain_vs_exact_rmsnorm(capi, consumer):
    """AFFINE_NORM producer -> SwiGLU / QKV consumer against the exact RMSNorm(h) * w * (1 + scale) + shift, @ W^T.
    The only approximations are bf16 roundings (out_scaled, the shift operand of ibias, the bf16 output: ~2^-9 relative
    each), so rel-L2 <= 5e-3."""
    g = gen(31)
    d, K0, T, items, eps = 512, 256, 250, 3, 1e-5
    M = T * items
    X = bf(randn(g, M, K0))
    W0 = bf(randn(g, d, K0, scale=K0 ** -0.5))
    res = randn(g, M, d)
    w_norm = 1 + 0.2 * randn(g, d)
    scale, shift = 0.2 * randn(g, items, d), 0.2 * randn(g, items, d)
    colscale = (w_norm * (1 + scale)).contiguous()
    h_bf = Out(M, d, torch.bfloat16)
    ssq = torch.full((M + 3, 4), SENT, device=DEV)      # the consumer reads rows of ssq_n = 4 partials: ld = 4
    launch(capi, linear_runs(K0, 64), mode=AFFINE_NORM, bn=256, bk=64, cg=1, a=X, a_cols=K0, a_rows=M, a_items=1, b=W0,
           n=d, res=res, res_ld=d, gate_div=T, colscale=colscale, colscale_ld=d, out_scaled=h_bf, ssq_out=ssq, ssq_ld=4)
    h_bf.assert_guards("out_scaled")
    assert (ssq[M:] == SENT).all() and (ssq[:M] > 0).all()
    N = 2 * 512 if consumer == "swiglu" else 3 * d
    W1 = bf(randn(g, N, d, scale=d ** -0.5))
    ibias = (bf(shift).double() @ W1.double().t()).float()
    out = Out(M, N // 2 if consumer == "swiglu" else N, torch.bfloat16)
    wq, wk = 1 + 0.3 * randn(g, 128), 1 + 0.3 * randn(g, 128)
    rope = rope_table(T, g)
    extra = dict(mode=QKV, qnorm_w=wq, knorm_w=wk, n_q_end=d, n_k_end=2 * d, rope=rope, rope_T=T, use_rope=1) \
        if consumer == "qkv" else dict(mode=SWIGLU)
    launch(capi, linear_runs(d, 64), bn=256, bk=64, cg=1, a=h_bf.buf, a_cols=d, a_rows=M, a_items=1, a_row_pitch=h_bf.ld,
           b=W1, n=N, out_bf16=out, ssq_in=ssq, ssq_n=4, ssq_inv_dim=1.0 / d, ibias=ibias, ibias_ld=N, ibias_div=T,
           eps=eps, **extra)
    out.assert_guards("consumer out")
    item = torch.arange(M, device=DEV) // T
    h = X.double() @ W0.double().t() + res.double()
    xn = h * (h.pow(2).mean(1, keepdim=True) + eps).rsqrt() * w_norm.double() * (1 + scale.double()[item]) \
        + shift.double()[item]
    y = xn @ W1.double().t()
    if consumer == "swiglu":
        y = y.view(M, N // 64, 2, 32)
        ref = (torch.nn.functional.silu(y[:, :, 0]) * y[:, :, 1]).reshape(M, N // 2)
    else:
        ref = qkv_ref(y, wq, wk, d, 2 * d, rope, torch.arange(M, device=DEV) % T, eps)
    err = rel_l2(out.val, ref)
    assert err < 5e-3, err


# ------------------------------------------------------------------------------------------------ schedule
SCHEDULES = [dict(grid_ctas=gc, group_m=gm, reverse_m=rv) for gc in ("default", "cg", "3cg") for gm in (0, 1, 5)
             for rv in (0, 1)]


@pytest.mark.parametrize("family", ["affine1", "affine2", "swiglu", "qkv", "xattn", "norm", "b2b", "transpose"])
def test_schedule_invariance_bit_exact(capi, family):
    """The same problem under every persistent-grid size (default, cg, 3 cg CTAs: many tiles per CTA, the stage ring
    wraps across tiles and the producer runs ahead into the next tile during the epilogue), group_m (default, 1, 5) and
    serpentine order gives bit-identical outputs; so do 1- and 2-CTA tiles at BN = 256 (same per-element k order)."""
    make = {
        "affine1": lambda cg: affine_case(capi, 256, 64, cg, T=250, items=5, seed=3),
        "affine2": lambda cg: affine_case(capi, 128, 32, cg, T=250, items=5, seed=4),
        "swiglu": lambda cg: swiglu_case(capi, cg, 1, seed=5),
        "qkv": lambda cg: qkv_case(capi, 256, cg, 1, 1, seed=6),
        "xattn": lambda cg: xattn_case(capi, 3, 3, cg=cg, seed=7),
        "norm": lambda cg: norm_producer_case(capi, cg, seed=8),
        "b2b": lambda cg: b2b_case(capi, 64, 64, seed=9),
        "transpose": lambda cg: conv_case(capi, "transpose", seed=10),
    }[family]
    cgs = (1, 2) if family in ("affine1", "swiglu", "qkv", "xattn", "norm") else (1,)
    base = None
    for cg in cgs:
        case = make(cg)
        for s in SCHEDULES:
            gc = {"default": 0, "cg": cg, "3cg": 3 * cg}[s["grid_ctas"]]
            got = case.run(grid_ctas=gc, group_m=s["group_m"], reverse_m=s["reverse_m"])
            if base is None:
                case.check(got)
                base = got
            for k in got:
                assert torch.equal(got[k], base[k]), (family, cg, s, k)


# ------------------------------------------------------------------------------------------------ debug switches
def _fresh_forward(m, inputs, env):
    """A new engine for `m` created and planned with the environment `env` (the switches are read at engine creation
    and at planning), then one DiT evaluation."""
    old = {k: os.environ.get(k) for k in env}
    try:
        for k, v in env.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
        if m._engine is not None:
            m._engine.close()
            m._engine = None
        m._ensure_engine()
        out = m.forward(**inputs)
        torch.cuda.synchronize()
        return out
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _eval_inputs(B, T, L, seed):
    from oracle import restate
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(B, T, 128, generator=g)
    sizes = torch.tensor([float(T - (T // 4) * (i % 3)) for i in range(B)])
    pad = restate.mask_from_sizes(sizes)
    ids, al = restate.process_anchors(None, pad, 1920, 48000)
    tmask = torch.ones(B, L, dtype=torch.bool)
    tmask[-1, max(1, L - 1):] = False
    return dict(noisy_audio=torch.randn(B, T, 256, generator=g).cuda(), audio_features=torch.cat([f, f], 2).cuda(),
                text_features=torch.randn(B, L, 768, generator=g).cuda(), time=torch.linspace(0.1, 0.9, B).cuda(),
                text_mask=tmask.cuda(), masked_video_features=torch.zeros(B, 1024, T).cuda(),
                anchor_ids=ids.cuda(), anchor_alignment=al.cuda(), audio_pad_mask=pad.cuda())


@pytest.fixture(scope="module", params=["tiny", "small"])
def switch_model(request):
    """(model, one evaluation's inputs): the tiny model (1-CTA tiles), and the small stand-in at B = 5 x T = 250
    (2-CTA cluster GEMMs, wgmma attention, fused cross-attention) with its weights kept on the GPU so that a fresh
    engine is cheap."""
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.synthetic import make_state_dict
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    name = "sam-audio-" + request.param
    cfg = stand_in_config(name)
    m = SAMAudio(cfg, text_encoder=SyntheticTextEncoder())
    m.load_state_dict(make_state_dict(cfg, seed=1))
    m = m.eval().cuda()
    m._state = {k: v.cuda() for k, v in m._state.items()}
    inputs = _eval_inputs(2, 29, 3, 41) if request.param == "tiny" else _eval_inputs(5, 250, 3, 42)
    yield m, inputs
    if m._engine is not None:
        m._engine.close()


SWITCHES_EXACT = ["SAB_FORCE_CG=1", "SAB_FORCE_CG=2", "SAB_NO_SERPENTINE=1"]
SWITCHES_APPROX = ["SAB_NO_FUSED_NORM=1", "SAB_NO_FUSED_XATTN=1", "SAB_NO_TC_ATTENTION=1"]
# rel-L2 of a switched DiT evaluation against the default path (the golden tolerance is 2e-2): the unfused RMSNorm
# rounds the normalised rows instead of h * w * (1 + scale), the streaming kernels round P and O differently.
# Measured on an H100 80GB HBM3, small stand-in at B = 5 x T = 250: 6.3e-4 (no fused norm), 7.2e-4 (no fused
# cross-attention), 5.4e-4 (no wgmma attention); the bound leaves 4x of that
SWITCH_BOUND = 3e-3


@pytest.mark.parametrize("switch", SWITCHES_EXACT + SWITCHES_APPROX)
def test_debug_switch_agrees_with_default(switch_model, switch):
    m, inputs = switch_model
    k, v = switch.split("=")
    off = {s.split("=")[0]: None for s in SWITCHES_EXACT + SWITCHES_APPROX + ["SAB_ATTN_POLY=0"]}
    ref = _fresh_forward(m, inputs, off)
    out = _fresh_forward(m, inputs, dict(off, **{k: v}))
    if switch in SWITCHES_EXACT:
        assert torch.equal(out, ref), (switch, rel_l2(out, ref))
    else:
        err = rel_l2(out, ref)
        print(f"[switch] {switch}: rel-L2 {err:.3e} vs default")
        assert 0 < err < SWITCH_BOUND, (switch, err)


def test_debug_switches_do_not_leak_into_later_engines(switch_model):
    """An engine created with SAB_FORCE_CG=1 and SAB_ATTN_POLY=0 must not change the engines created after the
    variables are removed: they give the default path's result bit for bit."""
    m, inputs = switch_model
    off = {"SAB_FORCE_CG": None, "SAB_ATTN_POLY": None}
    ref = _fresh_forward(m, inputs, off)
    forced = _fresh_forward(m, inputs, {"SAB_FORCE_CG": "1", "SAB_ATTN_POLY": "0"})
    assert not torch.equal(forced, ref)                 # the polynomial exponential changes the rounding
    again = _fresh_forward(m, inputs, off)
    assert torch.equal(again, ref), rel_l2(again, ref)


_DECODE = r"""
import sys, torch
sys.path.insert(0, sys.argv[1])
from sam_audio_b200.model import build_synthetic_model
m = build_synthetic_model("sam-audio-tiny", seed=0, device="cuda:0")
lat = torch.randn(3, 12, 256, generator=torch.Generator().manual_seed(5)).cuda()
out = torch.empty(3, 2, 12 * 1920, device="cuda")
m._ensure_engine().decode(lat, 3, 12, out)
torch.save(out.cpu(), sys.argv[2])
"""


def test_no_b2b_codec_decode_agrees(tiny_model, tmp_path):
    """SAB_NO_B2B is read once per process: a subprocess with it set decodes through the two-launch residual units,
    this process through the back-to-back ones.  Both round the intermediate Snake tile to bf16, so they differ only by
    fp32 summation order and __sinf rounding: rel-L2 <= 1e-3 (the codec's oracle tolerance is 3e-2)."""
    path = str(tmp_path / "decode_no_b2b.pt")
    env = dict(os.environ, SAB_NO_B2B="1")
    r = subprocess.run([sys.executable, "-c", _DECODE, ROOT, path], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    lat = torch.randn(3, 12, 256, generator=torch.Generator().manual_seed(5)).cuda()
    out = torch.empty(3, 2, 12 * 1920, device="cuda")
    tiny_model._ensure_engine().decode(lat, 3, 12, out)
    torch.cuda.synchronize()
    split = torch.load(path)
    err = rel_l2(out.cpu(), split)
    print(f"[switch] SAB_NO_B2B codec decode: rel-L2 {err:.3e}")
    assert err < 1e-3, err
