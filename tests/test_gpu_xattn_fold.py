"""The cross-attention output projection folded into the text values (sam_audio_b200/csrc/xattn_fold.cuh):

    cross.wo(O)[row, n] = sum_{h,j} P[row, j*H + h] * Ut[clip][n, j*H + h],   Ut[clip][n, j*H + h] = Wo[n, h-slice] . V[clip, j, h-slice]

Each piece is checked element-wise against float64 built from the bf16 operands the kernels read (bounds as in
test_gpu_gemm_epilogues.py): the fold kernel, the probabilities written by the fused cross.wq epilogue (xa_p), the
GEMM with a per-clip B operand (b_clip_rows / b_clip_div), and the three chained against Wo softmax(q K^T) V + h.
The engine's SAB_NO_XATTN_FOLD switch (the d x d cross.wo) is compared with the default.  The descriptor rules of the
new GemmParams fields are host-only tests.
"""
import math
import os

import pytest
import torch

from _util import rel_l2
from test_capi_exports import _FAKE, _XA, _gemm_desc, _gemm_ex_error, lib  # noqa: F401  (lib: module fixture)
from test_gpu_gemm_epilogues import (AFFINE, AFFINE_NORM, DEV, LOG2E, QKV, SCHEDULES, Case, Out, _fresh_forward,
                                     assert_close, bf, capi, gen, linear_runs, qkv_ref, randn,
                                     ref_acc, switch_model)  # noqa: F401  (capi, switch_model: fixtures)

gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ host-only rules
@pytest.mark.parametrize("fields,message", [
    (dict(b_clip_rows=256, b_clip_div=0), "b_clip_div=0 must be >= 1 with a per-clip B"),
    (dict(b_clip_rows=128, b_clip_div=1), "b_clip_rows=128 must be >= N=256"),
    (dict(b_clip_rows=-1, b_clip_div=1), "b_clip_rows=-1 must be >= 0"),
    (dict(xa_p=_FAKE, xa_p_ld=64), "xa_p (cross-attention probabilities) needs fused cross-attention"),
    (dict(_XA, out_bf16=None, xa_p=_FAKE, xa_p_ld=5), "xa_p_ld=5 is below heads * xa_Tk = 6"),
    (dict(_XA, bn=128, n=256, out_bf16=None, xa_p=_FAKE, xa_p_ld=8),
     "no GEMM instantiation for BN=128 BK=64 mode=2 cg=1 b2b=0 with xa_p"),
])
def test_fold_desc_rules_rejected(lib, fields, message):
    err = _gemm_ex_error(lib, _gemm_desc(**fields))
    assert err is not None and message in err, err


@pytest.mark.skipif(torch.cuda.is_available(), reason="the fake operands would reach the device")
def test_fold_desc_valid_passes_the_rules(lib):
    for fields in (dict(b_clip_rows=256, b_clip_div=3), dict(_XA, out_bf16=None, xa_p=_FAKE, xa_p_ld=8)):
        err = _gemm_ex_error(lib, _gemm_desc(**fields))
        assert err is not None and "sab_test_gemm_ex:" not in err, (fields, err)


# ------------------------------------------------------------------------------------------------ fold kernel
def fold(capi, wos, kv, kv_ld, d, L, clips, ldu, guard=64):
    """Run the fold for len(wos) layers; returns the raw buffer [layers * stride + guard] and the layer stride."""
    H = d // 128
    stride = clips * d * ldu + 256           # layer gap: must keep its sentinel
    ut = torch.full((len(wos) * stride + guard,), -7776.0, dtype=torch.bfloat16, device=DEV)
    tab = torch.tensor([w.data_ptr() for w in wos], dtype=torch.int64, device=DEV)
    capi.check(capi.lib().sab_test_xattn_fold(len(wos), clips, L, H, tab.data_ptr(), kv.data_ptr(), kv_ld, 2 * d, d,
                                              ut.data_ptr(), ldu, stride, capi.stream_ptr()))
    torch.cuda.synchronize()
    return ut, stride


def fold_ref(wo, v, clips, L, H):
    """fp64 Ut [clips, d, H*L] of one layer: wo [d, d], v [clips*L, d]."""
    d = H * 128
    w = wo.double().view(d, H, 128)
    vv = v.double().view(clips, L, H, 128)
    return torch.einsum("nhc,bjhc->bnjh", w, vv).reshape(clips, d, H * L)


@gpu
@pytest.mark.parametrize("L", [1, 3, 8])
def test_fold_kernel(capi, L):
    """Three layers from an all-layers K|V buffer; 40 clips so that the CTA sweeps several shared-memory chunks."""
    g = gen(100 + L)
    H, NL, clips = 10, 3, 40
    d = 128 * H
    ldu = (H * L + 7) // 8 * 8
    wos = [bf(randn(g, d, d, scale=d ** -0.5)) for _ in range(NL)]
    kv_ld = 2 * d * NL + 64
    kv = bf(randn(g, clips * L, kv_ld))
    ut, stride = fold(capi, wos, kv, kv_ld, d, L, clips, ldu)
    for l in range(NL):
        blk = ut[l * stride: l * stride + clips * d * ldu].view(clips, d, ldu)
        r = fold_ref(wos[l], kv[:, l * 2 * d + d: l * 2 * d + 2 * d], clips, L, H)
        assert_close(blk[:, :, : H * L].float(), r, f"fold layer {l}", bf16=True)
        assert (blk[:, :, H * L:].float() == 0).all(), "padding columns must be 0"
        gap = ut[l * stride + clips * d * ldu: (l + 1) * stride].float()
        assert (gap == -7776.0).all(), f"writes past layer {l}"
    assert (ut[NL * stride:].float() == -7776.0).all()


# ------------------------------------------------------------------------------------------------ probabilities
def xattn_p_case(capi, Tk, cand, cg=1, seed=0):
    """The fused cross.wq epilogue with xa_p: each row's normalised probabilities at column j * H + h."""
    g = gen(seed)
    d, K, T, B_clips, NL = 384, 256, 100, 2, 3
    H, M = d // 128, B_clips * cand * T
    A = bf(randn(g, M, K))
    W = bf(randn(g, d, K, scale=K ** -0.5))
    wq = 1 + 0.3 * randn(g, 128)
    kv_ld = 2 * d * NL
    kv = bf(randn(g, B_clips * Tk, kv_ld))
    kv_l = kv[:, 2 * d: 4 * d]
    mask = torch.ones(B_clips, Tk, dtype=torch.uint8, device=DEV)
    mask[1, max(1, Tk - 2):] = 0
    out = Out(M, H * Tk, torch.bfloat16)
    fields = dict(mode=QKV, bn=256, bk=64, cg=cg, a=A, a_cols=K, a_rows=M, a_items=1, b=W, n=d, xa_p=out,
                  qnorm_w=wq, knorm_w=wq, n_q_end=d, n_k_end=d, rope_T=T, eps=1e-5,
                  xa_kv=kv.data_ptr() + 2 * d * 2, xa_kv_ld=kv_ld, xa_v_col0=d, xa_Tk=Tk, xa_T=T * cand, xa_mask=mask,
                  xa_scale_log2=LOG2E / math.sqrt(128))
    runs = linear_runs(K, 64)
    clip = torch.arange(M, device=DEV) // (T * cand)

    def probs():
        q = qkv_ref(ref_acc(A.view(1, M, K), W, runs, 64), wq, wq, d, d, None, None, 1e-5)
        Kt = kv_l[:, :d].double().contiguous().view(B_clips, Tk, H, 128)[clip]
        s = torch.einsum("mhc,mjhc->mhj", q.view(M, H, 128), Kt) / math.sqrt(128)
        s = s.masked_fill(~mask.bool()[clip][:, None, :], float("-inf"))
        return torch.softmax(s, -1).transpose(1, 2)                            # [M, Tk, H]

    def check(got):
        p = got["xa_p"].view(M, Tk, H)
        masked = ~mask.bool()[clip][:, :, None].expand(M, Tk, H)
        assert (p[masked] == 0).all(), "masked tokens must give exact zeros"
        assert_close(got["xa_p"], probs().reshape(M, Tk * H), "cross-attention probabilities", bf16=True)
    c = Case(capi, runs, fields, {"xa_p": out}, check)
    c.probs, c.kv_l, c.mask, c.M, c.H, c.d, c.T, c.B_clips = probs, kv_l, mask, M, H, d, T, B_clips
    return c


@gpu
@pytest.mark.parametrize("cand", [1, 3])
@pytest.mark.parametrize("Tk", [1, 3, 8])
def test_cross_attention_probabilities(capi, Tk, cand):
    c = xattn_p_case(capi, Tk, cand, seed=200 + Tk + 10 * cand)
    c.check(c.run())


# ------------------------------------------------------------------------------------------------ per-clip B GEMM
def per_clip_case(capi, mode, cg, cand, seed=0, T=250, clips=2, H=3, L=3, N=512):
    """cross.wo as the engine plans it: A = P [items = clips*cand, T, H*L] (pitch ldu, TMA zero-fills the k-block),
    B = Ut [clips * N, H*L] (pitch ldu, per clip), in-place style residual, fp32 out; AFFINE_NORM adds the fused-norm
    producer outputs."""
    g = gen(seed)
    K, items = H * L, clips * cand
    ldu = (K + 7) // 8 * 8
    M = items * T
    Ab = torch.zeros(M, ldu, device=DEV, dtype=torch.bfloat16)
    Ab[:, :K] = bf(torch.rand(M, K, device=DEV, generator=g))
    Bb = torch.zeros(clips * N, ldu, device=DEV, dtype=torch.bfloat16)
    Bb[:, :K] = bf(randn(g, clips * N, K))
    Ab[:, K:] = float("nan")                 # past the visible width: must never be read
    Bb[:, K:] = float("nan")
    res = randn(g, M, N)
    out = Out(M, N, torch.float32)
    outs = {"out_f32": out}
    fields = dict(mode=mode, bn=256, bk=64, cg=cg, a=Ab, a_cols=K, a_rows=T, a_items=items, a_row_pitch=ldu,
                  a_item_pitch=T * ldu, b=Bb, n=N, b_cols=K, b_ld=ldu, b_clip_rows=N, b_clip_div=cand,
                  res=res, res_ld=N, out_f32=out)
    if mode == AFFINE_NORM:
        colscale = 1 + 0.2 * randn(g, items, N)
        sc, ssq = Out(M, N, torch.bfloat16), Out(M, 2 * (N // 256), torch.float32)
        fields.update(out_scaled=sc, colscale=colscale, colscale_ld=N, gate_div=T, ssq_out=ssq)
        outs.update(out_scaled=sc, ssq_out=ssq)
    runs = [[(0, 0, (K + 63) // 64)]]

    def check(got):
        clip = torch.arange(M, device=DEV) // (T * cand)
        Bc = Bb[:, :K].double().view(clips, N, K)[clip]                       # [M, N, K]
        v = torch.einsum("mk,mnk->mn", Ab[:, :K].double(), Bc) + res.double()
        assert_close(got["out_f32"], v, "per-clip B affine")
        if mode == AFFINE_NORM:
            item = torch.arange(M, device=DEV) // T
            assert_close(got["out_scaled"], v * colscale.double()[item], "per-clip B out_scaled", bf16=True)
            s = (v * v).view(M, N // 256, 8, 32).sum(-1)
            ref_ssq = torch.stack([s[:, :, 0::2].sum(-1), s[:, :, 1::2].sum(-1)], -1).reshape(M, -1)
            assert_close(got["ssq_out"], ref_ssq, "per-clip B ssq")
    return Case(capi, runs, fields, outs, check)


@gpu
@pytest.mark.parametrize("cand", [1, 3])
@pytest.mark.parametrize("cg", [1, 2])
@pytest.mark.parametrize("mode", [AFFINE, AFFINE_NORM])
def test_per_clip_b_gemm(capi, mode, cg, cand):
    c = per_clip_case(capi, mode, cg, cand, seed=300 + 10 * cg + cand + mode)
    c.check(c.run())


@gpu
@pytest.mark.parametrize("mode", [AFFINE, AFFINE_NORM])
def test_per_clip_b_schedule_invariance_bit_exact(capi, mode):
    """Grid size, group_m, serpentine order and 1- vs 2-CTA tiles give bit-identical per-clip results."""
    base = None
    for cg in (1, 2):
        case = per_clip_case(capi, mode, cg, 3, seed=400 + mode)
        for s in SCHEDULES:
            gc = {"default": 0, "cg": cg, "3cg": 3 * cg}[s["grid_ctas"]]
            got = case.run(grid_ctas=gc, group_m=s["group_m"], reverse_m=s["reverse_m"])
            if base is None:
                case.check(got)
                base = got
            for k in got:
                assert torch.equal(got[k], base[k]), (mode, cg, s, k)


# ------------------------------------------------------------------------------------------------ the whole identity
@gpu
@pytest.mark.parametrize("cand", [1, 3])
def test_probabilities_fold_gemm_equal_output_projection(capi, cand):
    """P from the cross.wq epilogue, Ut from the fold, then the per-clip GEMM with the residual: against
    h + Wo softmax(q K^T) V in float64.  Bound: the bf16 roundings of P and Ut, 2^-7 sum |P| |Ut|, on top of the usual
    1e-3 rms_row term."""
    Tk = 3
    c = xattn_p_case(capi, Tk, cand, seed=500 + cand)
    got_p = c.run()["xa_p"]                                   # [M, H*Tk] bf16
    M, H, d, T, B_clips = c.M, c.H, c.d, c.T, c.B_clips
    g = gen(600 + cand)
    wo = bf(randn(g, d, d, scale=d ** -0.5))
    ldu = (H * Tk + 7) // 8 * 8
    ut, _ = fold(capi, [wo], c.kv_l.contiguous(), 2 * d, d, Tk, B_clips, ldu)
    Ut = ut[: B_clips * d * ldu].view(B_clips * d, ldu)
    Pb = torch.zeros(M, ldu, device=DEV, dtype=torch.bfloat16)
    Pb[:, : H * Tk] = got_p
    h = randn(g, M, d)
    out = Out(M, d, torch.float32)
    from test_gpu_gemm_epilogues import launch
    launch(capi, [[(0, 0, 1)]], mode=AFFINE, bn=256, bk=64, cg=0, a=Pb, a_cols=H * Tk, a_rows=T * cand,
           a_items=B_clips, a_row_pitch=ldu, a_item_pitch=T * cand * ldu, b=Ut, n=d, b_cols=H * Tk, b_ld=ldu,
           b_clip_rows=d, b_clip_div=1, res=h, res_ld=d, out_f32=out)
    out.assert_guards("out_f32")
    clip = torch.arange(M, device=DEV) // (T * cand)
    Vt = c.kv_l[:, d:].double().contiguous().view(B_clips, Tk, H, 128)[clip]
    o = torch.einsum("mjh,mjhc->mhc", c.probs(), Vt).reshape(M, d)
    ref = h.double() + o @ wo.double().t()
    Ud = Ut[:, : H * Tk].double().view(B_clips, d, H * Tk)[clip]
    extra = 2.0 ** -7 * torch.einsum("mk,mnk->mn", got_p.double().abs(), Ud.abs())
    assert_close(out.val, ref, "P -> fold -> per-clip GEMM", extra=extra, rms=(o @ wo.double().t()).pow(2).mean(-1, keepdim=True).sqrt())


# ------------------------------------------------------------------------------------------------ engine switch
FOLD_BOUND = 3e-3     # the bound every approximate debug switch is held to (test_gpu_gemm_epilogues.SWITCH_BOUND)


@gpu
def test_no_xattn_fold_switch_agrees_with_default(switch_model):
    m, inputs = switch_model
    off = {"SAB_NO_XATTN_FOLD": None, "SAB_NO_FUSED_XATTN": None}
    ref = _fresh_forward(m, inputs, off)
    out = _fresh_forward(m, inputs, dict(off, SAB_NO_XATTN_FOLD="1"))
    err = rel_l2(out, ref)
    print(f"[switch] SAB_NO_XATTN_FOLD=1: rel-L2 {err:.3e} vs default")
    assert 0 < err < FOLD_BOUND, err
    unfused = _fresh_forward(m, inputs, dict(off, SAB_NO_FUSED_XATTN="1"))
    err2 = rel_l2(unfused, ref)
    print(f"[switch] SAB_NO_FUSED_XATTN=1: rel-L2 {err2:.3e} vs default (fold)")
    assert 0 < err2 < FOLD_BOUND, err2
    again = _fresh_forward(m, inputs, off)                    # the switch does not outlive its engine
    assert torch.equal(again, ref), rel_l2(again, ref)


def _fresh_solve(m, inputs, env, cand, noise):
    """A new engine with the environment `env`, conditioning for `cand` candidates per clip, one midpoint step."""
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
        eng = m._ensure_engine()
        with torch.inference_mode():
            m._install_conditioning(inputs["audio_features"], inputs["text_features"], inputs["text_mask"],
                                    inputs["masked_video_features"], inputs["anchor_ids"], inputs["anchor_alignment"],
                                    inputs["audio_pad_mask"], candidates=cand)
            latent = torch.empty_like(noise)
            with torch.cuda.device(noise.device):
                eng.solve(noise, 1, latent, "midpoint")
        torch.cuda.synchronize()
        return latent
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


@gpu
def test_no_xattn_fold_switch_with_candidates(switch_model):
    """Two candidates per clip share the clip's Ut: the velocity of one midpoint step agrees with the d x d path."""
    m, inputs = switch_model
    B, T = inputs["audio_features"].shape[:2]
    noise = torch.randn(B * 2, T, 256, generator=torch.Generator().manual_seed(7)).cuda()
    ref = _fresh_solve(m, inputs, {"SAB_NO_XATTN_FOLD": None}, 2, noise)
    out = _fresh_solve(m, inputs, {"SAB_NO_XATTN_FOLD": "1"}, 2, noise)
    err = rel_l2(out - noise, ref - noise)
    print(f"[switch] SAB_NO_XATTN_FOLD=1, 2 candidates: rel-L2 {err:.3e} vs default")
    assert 0 < err < FOLD_BOUND, err
