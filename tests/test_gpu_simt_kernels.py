"""GPU (H100): the SIMT kernels of the DiT, codec and T5 paths one at a time, through the sab_test_* seams (each launches
the engine's own launch helper: same kernels, grids and variant choice), element by element against float64 computed
from exactly the operands the kernel reads (bf16 operands upcast exactly).  The argument rules of the seams are checked
host-only at the end of the file (no GPU needed).

Bounds, per element, with r the float64 reference:
  * bf16 outputs ....................... |o - r| <= 2^-8 |r| + tau s    (round to nearest: half an ulp <= 2^-8 |r|)
    s is the element's magnitude scale and tau covers the kernel's fp32 arithmetic:
      rmsnorm_mod   s = |x rstd w (1 + scale)| + |shift|, tau = 1e-5 (fp32 row sum of squares over d <= 4096, rsqrtf)
      GN + SiLU     s = |z - beta| + |beta| with tau = 1e-5 (fp32 per-thread partials, __expf / rcp.approx SiLU), plus
                    2^-21 |gamma| rstd (|x| + |mean|): the fp32 roundings of the mean and of x - mean
      t5_norm       s = |x rstd w|, tau = 1e-5
      time features s = 1, tau = 2^-20, plus 2^-21 |argument| (expf / cosf / sinf: a few fp32 ulps of the phase)
      xattn_small   s = sum_j p_j |v_j|, tau = 1e-4 (fp32 scores and ex2.approx probabilities, P kept in fp32)
      t5_attention  s = sum_j p_j |v_j|, tau = 1e-4 (fp32 scores, __expf, fp32 sums over up to 512 keys)
  * fp32 outputs ....................... |o - r| <= tau s with the same scales (ln_vector, cond_finish, t5_norm fp32,
    enc.conv0's x_out: s = |bias| + sum_k |w x|, tau = 2^-21 for 7 FMAs; the anchor table: s = sum_k |a b|,
    tau = K 2^-24); cond_finish's near-constant video rows also carry the fp32 error of the row mean,
    rstd (d/32 + 5) 2^-24 mean|x| (per-lane sums of d/32 terms, then a 5-level shuffle tree), times |w gate|
  * dec.last (tanh of a 7 x C dot product): |o - r| <= (1 - r^2) 2^-24 (7 C) sum |w a| + 2^-22
  * Snake (enc.conv0's a_out): the Snake bound of _util.snake_bound on the kernel's own x_out, plus the bf16 rounding
  * rope_table: |o - r| <= 2^-22 |pos inv| + 2^-22 against float64 and against the reference's own fp32 formula
  * attention_kernel (Tk > 16, P rounded to bf16): rel-L2 <= 1e-2 as for the other attention kernels
  * build_mod / norm_tables: bit-exact (one fp32 add or multiply, a bf16 cast) against torch on the same operands
Systematic-error check: a per-element bf16 bound cannot see a relative error below 2^-9 (a wrong divisor in a mean, a
wrong eps).  For the bf16 normalisations (rmsnorm_mod, GN + SiLU, t5_norm) the mean signed error, in ulps of r and signed
along the direction a too large rstd would move the element, must be near zero: round-to-nearest is unbiased.  It is
taken over the elements whose fp32 error budget (the tau s terms above) is below 1/16 ulp, where the error is the rounding
alone, and must stay within SYS_FLOOR + 6 sigma, sigma = 0.29 / sqrt(n) the spread of the mean of n uniform roundings.
Calibration on an H100 80GB HBM3 (700 W) with the kernels as committed: every |bias| is within 2 sigma of zero except
on the GN + SiLU slabs of millions of elements, where a real bias of up to 6.2e-4 ulp shows (mean / std = 300, 3.9 M
elements; the SiLU's approximate exponential and reciprocal).  SYS_FLOOR = 3e-3 is about 5x that.  A divisor of d - 1
instead of d at d = 4096 scales rstd by 1 - 1.2e-4, which moves the bias by about 1.2e-4 |r| / ulp(r) = 2e-2 ulp.
cond_finish writes fp32, whose kernel arithmetic (not a rounding) dominates each element's error; there the check is the
least-squares relative scale of the LayerNorm term, sum((o - r) t) / sum(t^2) with t = tanh(g_v) LayerNorm(v) w,
within SYS_SCALE = 1e-5 (measured -8.2e-8 on the same H100; a divisor of d - 1 moves it by 1 / (2d) = 6.5e-4).
Every output lives in a sentinel-filled buffer with guard elements before and after it that must survive, and every
output must be finite.
"""
import math

import pytest
import torch

from _util import rel_l2, snake_bound

SENT = -7776.0            # exactly representable in bf16 and fp32
DEV = "cuda"
G = 64                    # guard elements on each side (keeps 16-byte alignment for fp32 and bf16)
SYS_FLOOR = 3e-3          # bf16 systematic-error floor, ulps (module docstring)
SYS_SCALE = 1e-5          # cond_finish LayerNorm relative scale error
_FAKE = 1 << 20           # a 16 B aligned non-null address for the host-only rejection cases

gpu = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    return _capi


# ------------------------------------------------------------------------------------------------ helpers
class Buf:
    """An output of `n` elements (viewed as `shape`) inside a sentinel-filled buffer with G guard elements each side."""

    def __init__(self, shape, dtype):
        self.shape = tuple(shape)
        self.n = math.prod(self.shape)
        self.buf = torch.full((self.n + 2 * G,), SENT, dtype=dtype, device=DEV)

    @property
    def ptr(self):
        return self.buf.data_ptr() + G * self.buf.element_size()

    @property
    def val(self):
        return self.buf[G: G + self.n].view(self.shape)

    def check(self, what):
        torch.cuda.synchronize()
        guards = torch.cat([self.buf[:G], self.buf[G + self.n:]]).float()
        assert bool((guards == SENT).all()), f"{what}: {int((guards != SENT).sum())} writes outside the output"
        assert bool(torch.isfinite(self.val.float()).all()), f"{what}: non-finite or unwritten outputs"
        return self.val


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def randn(g, *shape, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=g) * scale


def assert_bound(o, r, tol, what):
    err = (o.double() - r.double()).abs()
    bad = err > tol
    if bool(bad.any()):
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bound; first at flat index {i}: "
                             f"got {float(o.flatten()[i])}, want {float(r.flatten()[i])}, bound {float(tol.flatten()[i])}; "
                             f"max err/bound {float((err / tol).max()):.3g}")


def ulp(r, mant_bits):
    """ulp of r in a format with `mant_bits` stored mantissa bits (7: bf16, 23: fp32)."""
    _, e = torch.frexp(r.double())
    return torch.ldexp(torch.ones_like(r, dtype=torch.float64), (e - 1 - mant_bits).to(torch.int32))


def systematic(o, r, direction, arith, what):
    """Mean signed error of a bf16 output in ulps of r, signed along `direction` (where a too large rstd moves the
    element), over the elements whose fp32 error budget `arith` is below 1/16 ulp (there the error is the rounding
    alone, uniform in [-1/2, 1/2] ulp: standard deviation 0.29 / sqrt(n) for the mean of n)."""
    r = r.double()
    u = ulp(r, 7)
    keep = (r != 0) & (direction != 0) & (arith <= u / 16)
    e = ((o.double() - r) / u * torch.sign(direction))[keep]
    n = e.numel()
    if n < 1000:                       # too few roundings for a mean to mean anything (the T = 1, C = 64 slabs)
        return
    bias, limit = float(e.mean()), SYS_FLOOR + 6 * 0.29 / math.sqrt(n)
    print(f"[systematic] {what}: {bias:+.3e} ulp over {n} elements (limit {limit:.2e})")
    assert abs(bias) <= limit, f"{what}: mean signed error {bias:+.3e} ulp (limit {limit:.2e}): a systematic error"


def systematic_scale(o, r, t, what):
    """Least-squares relative scale error of the term t inside an fp32 output: sum((o - r) t) / sum(t^2).  A wrong
    rstd by a factor 1 + delta gives delta; the fp32 roundings average out."""
    a = float(((o.double() - r) * t).sum() / (t * t).sum())
    print(f"[systematic] {what}: relative scale error {a:+.3e} (limit {SYS_SCALE:.0e})")
    assert abs(a) <= SYS_SCALE, f"{what}: relative scale error {a:+.3e} (limit {SYS_SCALE:.0e}): a systematic error"


def bf(x):
    return x.bfloat16()


# ------------------------------------------------------------------------------------------------ rmsnorm_mod
RMS_DIMS = [256, 512, 1024, 1536, 2048, 2560, 2816, 3072, 4096]     # d / 128 = 2, 4, 8, 12, 16, 20, 22, 24, 32


def run_rmsnorm(capi, x, w, shift, scale, mod_ld, rows_per_item, eps, reverse):
    M, d = x.shape
    out = Buf((M, d), torch.bfloat16)
    capi.check(capi.lib().sab_test_rmsnorm_mod(M, d, x.data_ptr(), w.data_ptr(), shift.data_ptr(), scale.data_ptr(),
                                               mod_ld, rows_per_item, eps, reverse, out.ptr, capi.stream_ptr()))
    return out.check(f"rmsnorm_mod d={d}").clone()


def rmsnorm_case(d, M, rows_per_item, shared, seed):
    g = gen(seed)
    row_scale = torch.exp(randn(g, M, 1, scale=2.0))                # rows of very different scale
    x = randn(g, M, d) * row_scale
    x[1] *= 1e-4                                                      # mean(x^2) ~ 1e-8 << eps: eps dominates
    x[M // 2] = 1e-3 * randn(g, d)
    w = 1 + 0.2 * randn(g, d)
    n_items = (M + rows_per_item - 1) // rows_per_item
    mod = randn(g, 1 if shared else n_items, 6, d, scale=0.3)        # the adaLN row block [6, d] of each item
    return x, w, mod


@gpu
@pytest.mark.parametrize("d", RMS_DIMS)
def test_rmsnorm_mod_every_instantiation(capi, d):
    """Every rmsnorm_mod_kernel<d/128> instantiation, M not a multiple of 8, per-item rows (mod_ld = 6d) and shared rows
    (mod_ld = 0), forward and reverse row order bit-identical, rows of very different scale including ones where eps
    dominates; element bound and systematic-error check."""
    eps = 1e-5
    for M, rows_per_item, shared in ((203, 50, False), (77, 77, True), (9, 1, False)):
        x, w, mod = rmsnorm_case(d, M, rows_per_item, shared, seed=d + M)
        shift, scale = mod[:, 0], mod[:, 1]                           # rows 0 / 1 of the item's [6, d] block
        mod_ld = 0 if shared else 6 * d
        o = run_rmsnorm(capi, x, w, shift, scale, mod_ld, rows_per_item, eps, 0)
        o_rev = run_rmsnorm(capi, x, w, shift, scale, mod_ld, rows_per_item, eps, 1)
        assert torch.equal(o.view(torch.int16), o_rev.view(torch.int16)), f"d={d} M={M}: reverse order changed bits"
        b = torch.arange(M, device=DEV) // rows_per_item
        if shared:
            b = torch.zeros_like(b)
        xd = x.double()
        rstd = torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps)
        nt = xd * rstd * w.double() * (1 + scale.double()[b])
        r = nt + shift.double()[b]
        arith = 1e-5 * (nt.abs() + shift.double()[b].abs())
        assert_bound(o, r, 2.0 ** -8 * r.abs() + arith, f"rmsnorm_mod d={d} M={M} rows_per_item={rows_per_item}")
        systematic(o, r, nt, arith, f"rmsnorm_mod d={d} M={M}")


# ------------------------------------------------------------------------------------------------ GroupNorm + SiLU
def gn_ref(x, gamma, beta, eps, C):
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    var = (xd - mean).pow(2).mean(-1, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    gm = gamma.double().repeat(x.shape[1] // C).view(1, -1)
    bt = beta.double().repeat(x.shape[1] // C).view(1, -1)
    z = (xd - mean) * rstd * gm + bt
    y = z * torch.sigmoid(z)
    sig = torch.sigmoid(z)
    dsilu = sig * (1 + z * (1 - sig))
    arith = 1e-5 * ((z - bt).abs() + bt.abs()) + 2.0 ** -21 * gm.abs() * rstd * (xd.abs() + mean.abs())
    return y, arith, dsilu * (z - bt)


@gpu
@pytest.mark.parametrize("T,C,items", [(1, 64, 2), (1, 2816, 2), (250, 1024, 3), (10000, 2816, 1)])
@pytest.mark.parametrize("offset", [0.0, 1.0, 30.0, 300.0])
def test_group_norm_silu(capi, T, C, items, offset):
    """GN(1 group) + SiLU over whole (T, C) slabs: T = 1 (C = 64 leaves chunks with empty ranges), T = 250, and one
    28 M-element item (T = 10000, d = 2816); inputs with mean / std in {0, 1, 30, 300}; per-channel affine."""
    g = gen(T + C + int(offset))
    n = T * C
    x = randn(g, items, n)
    x += offset * (1 + 0.1 * torch.arange(items, device=DEV).view(-1, 1))   # a different DC offset per item
    gamma = 1 + 0.3 * randn(g, C)
    beta = 0.3 * randn(g, C)
    y = Buf((items, n), torch.bfloat16)
    capi.check(capi.lib().sab_test_group_norm_silu(items, n, C, x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), 1e-5,
                                                   y.ptr, capi.stream_ptr()))
    o = y.check(f"gn_silu T={T}")
    r, arith, direction = gn_ref(x, gamma, beta, 1e-5, C)
    del x
    assert_bound(o, r, 2.0 ** -8 * r.abs() + arith, f"gn_silu T={T} C={C} mean/std={offset}")
    systematic(o, r, direction, arith, f"gn_silu T={T} C={C} mean/std={offset}")


# ------------------------------------------------------------------------------------------------ cross-attention
def attn_ref(q, k, v, mask, items, heads, Tq, Tk, cand):
    """float64 softmax(Q K^T / sqrt(128) + mask) V, the cand query items of a clip sharing its K / V / mask."""
    qd = q.double().view(items, Tq, heads, 128).transpose(1, 2)
    kd = k.double().view(items // cand, Tk, heads, 128).transpose(1, 2).repeat_interleave(cand, 0)
    vd = v.double().view(items // cand, Tk, heads, 128).transpose(1, 2).repeat_interleave(cand, 0)
    s = qd @ kd.transpose(-1, -2) / math.sqrt(128.0)
    m = mask.bool().repeat_interleave(cand, 0)[:, None, None, :]
    p = torch.softmax(s.masked_fill(~m, float("-inf")), -1)
    o = (p @ vd).transpose(1, 2).reshape(items * Tq, heads * 128)
    mag = (p @ vd.abs()).transpose(1, 2).reshape(items * Tq, heads * 128)
    return o, mag


@gpu
@pytest.mark.parametrize("cand", [1, 3])
@pytest.mark.parametrize("Tq", [1, 127, 250, 300])
def test_attention_cross_dispatcher(capi, Tq, cand):
    """The engine's cross-attention dispatcher at every xattn_small bucket edge and past it (Tk = 1, 4 | 5, 8 | 9,
    15, 16 | 17, 20), ragged text masks that differ per clip, the candidates of a clip sharing its text (kv_div =
    mask_div = cand).  xattn_small keeps P in fp32: element bound; attention_kernel rounds P to bf16: rel-L2."""
    heads, clips = 2, 2
    items = clips * cand
    for Tk in (1, 4, 5, 8, 9, 15, 16, 17, 20):
        g = gen(Tq * 100 + Tk * 10 + cand)
        q = bf(randn(g, items * Tq, heads * 128, scale=1.5))
        k = bf(randn(g, clips * Tk, heads * 128))
        v = bf(randn(g, clips * Tk, heads * 128))
        mask = torch.ones(clips, Tk, dtype=torch.uint8, device=DEV)
        for c in range(clips):                                       # clip c keeps its first Tk - 2c keys (>= 1)
            mask[c, max(1, Tk - 2 * c - (Tk // 3) * c):] = 0
        if Tk > 2:
            mask[0, 1] = 0                                           # a hole, not only a ragged end
        o = Buf((items * Tq, heads * 128), torch.bfloat16)
        capi.check(capi.lib().sab_test_attention_cross(items, heads, Tq, Tk, cand, q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                       mask.data_ptr(), o.ptr, capi.stream_ptr()))
        out = o.check(f"attention_cross Tk={Tk}")
        r, mag = attn_ref(q, k, v, mask, items, heads, Tq, Tk, cand)
        what = f"attention_cross Tq={Tq} Tk={Tk} cand={cand}"
        if Tk <= 16:
            assert_bound(out, r, 2.0 ** -8 * r.abs() + 1e-4 * mag, what)
        else:
            assert rel_l2(out, r) <= 1e-2, what


# ------------------------------------------------------------------------------------------------ conditioning finish
def ln_ref(x, w, b, eps=1e-5):
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = torch.rsqrt((xd - mean).pow(2).mean(-1, keepdim=True) + eps)
    nt = (xd - mean) * rstd * w.double()
    return nt + b.double(), nt, mean, rstd


@gpu
@pytest.mark.parametrize("cand", [1, 4])
@pytest.mark.parametrize("mode", ["video", "absent_video", "no_video_term", "no_anchors"])
def test_cond_finish(capi, cand, mode):
    """sab_prepare's conditioning finish: LayerNorm of the projected video rows (including near-constant rows of variance
    ~1e-6, where eps = 1e-5 dominates), the constant vector for absent video (LayerNorm of the conv bias), the anchor table
    and its gather with more than 64 anchor ids per clip, SAB_PREP_NO_VIDEO_TERM / SAB_PREP_NO_ANCHORS; with candidates
    each candidate row equals its clip row."""
    B, T, d, n_anchor, adim, n_ids = 2, 51, 768, 4, 128, 80
    g = gen(cand * 7 + len(mode))
    cond_clip = randn(g, B * T, d)
    vproj = randn(g, B * T, d) * torch.exp(randn(g, B * T, 1)) + 3 * randn(g, B * T, 1)
    vproj[5] = 2.5 + 1e-3 * randn(g, d)                               # near-constant rows
    vproj[T + 7] = -4.0 + 1e-3 * randn(g, d)
    ln_w, ln_b = 1 + 0.2 * randn(g, d), 0.1 * randn(g, d)
    vid_bias = 0.5 + randn(g, d)
    gate_v, gate_a = torch.tensor([0.7], device=DEV), torch.tensor([-0.4], device=DEV)
    emb, proj = randn(g, n_anchor, adim), randn(g, d, adim, scale=adim ** -0.5)
    ids = torch.randint(0, n_anchor, (B, n_ids), device=DEV, generator=g)
    align = torch.randint(0, n_ids, (B, T), device=DEV, generator=g)
    align[0, :3] = torch.tensor([64, 70, 79], device=DEV)             # slots beyond 64
    flags = {"video": 0, "absent_video": 0, "no_video_term": 1, "no_anchors": 2}[mode]
    M = B * cand * T
    cond = Buf((M, d), torch.float32)
    if cand == 1:
        cond.val.copy_(cond_clip)                                      # in place, as the engine runs it
    clip_ptr = cond.ptr if cand == 1 else cond_clip.data_ptr()
    vconst, table = Buf((d,), torch.float32), Buf((n_anchor, d), torch.float32)
    capi.check(capi.lib().sab_test_cond_finish(
        B, cand, T, d, cond.ptr, clip_ptr, vproj.data_ptr() if mode == "video" else None, ln_w.data_ptr(), ln_b.data_ptr(),
        vid_bias.data_ptr(), vconst.ptr, gate_v.data_ptr(), emb.data_ptr(), proj.data_ptr(), n_anchor, adim, table.ptr,
        None if mode == "no_anchors" else ids.data_ptr(), n_ids, None if mode == "no_anchors" else align.data_ptr(),
        gate_a.data_ptr(), flags, capi.stream_ptr()))
    out, vc, tab = cond.check("cond"), vconst.check("vconst"), table.check("anchor_table")
    # the load-time tables against float64
    r_vc, nt_vc, _, _ = ln_ref(vid_bias, ln_w, ln_b)
    assert_bound(vc, r_vc, 1e-5 * (nt_vc.abs() + ln_b.double().abs()), "ln_vector")
    r_tab = emb.double() @ proj.double().t()
    assert_bound(tab, r_tab, adim * 2.0 ** -24 * (emb.double().abs() @ proj.double().abs().t()), "small_abt")
    # cond against float64 from the operands cond_finish reads (its own vconst / anchor table)
    gv = math.tanh(0.7) if mode != "no_video_term" else 0.0
    ga = math.tanh(-0.4) if mode != "no_anchors" else 0.0
    ci = cond_clip.double()
    s = ci.abs()
    r = ci.clone()
    nt_dir = None
    if mode == "video":
        vt, nt, mean, rstd = ln_ref(vproj, ln_w, ln_b)
        r += gv * vt
        e_mean = (d / 32 + 5) * 2.0 ** -24 * vproj.double().abs().mean(-1, keepdim=True)
        s += abs(gv) * (nt.abs() + ln_b.double().abs())
        extra = abs(gv) * ln_w.double().abs() * rstd * (e_mean + 2.0 ** -23 * (vproj.double() - mean).abs())
        nt_dir = gv * nt
    else:
        vcd = vc.double().view(1, d)
        r += gv * vcd
        s += abs(gv) * vcd.abs()
        extra = torch.zeros_like(r)
    if ga != 0.0:
        er = tab.double()[ids.gather(1, align).view(-1)]
        r += ga * er
        s += abs(ga) * er.abs()
    rows = torch.arange(M, device=DEV)
    crow = (rows // T // cand) * T + rows % T                         # the clip row of each sequence row
    r, s, extra = r[crow], s[crow], extra[crow] if mode == "video" else 0.0
    assert_bound(out, r, 1e-5 * s + extra, f"cond_finish {mode} cand={cand}")
    if cand > 1:
        per = out.view(B, cand, T, d)
        assert all(torch.equal(per[:, 0], per[:, j]) for j in range(cand)), "candidate rows differ from their clip row"
    if nt_dir is not None:
        systematic_scale(out, r, nt_dir[crow], f"cond_finish LayerNorm cand={cand}")


# ------------------------------------------------------------------------------------------------ time features
TIMES = [0.0, 1 / 32, 0.5, 31 / 32, 1.0]


@gpu
def test_time_features(capi):
    """tfreq and mem_time (cos | sin of t * exp(-ln(1e4) k / half)) at t = 0, 1/32, 0.5, 31/32, 1, with 3 candidates per
    clip whose times differ (the clip's text memory takes its first candidate's time)."""
    cand, clips, d, L = 3, 5, 256, 7
    R = cand * clips
    time = torch.tensor([TIMES[(i // cand) % 5] + (i % cand) * 0.01 for i in range(R)], device=DEV)
    g = gen(11)
    mem_base = randn(g, clips * L, d)
    tfreq, mem_in = Buf((R, 256), torch.bfloat16), Buf((clips * L, d), torch.bfloat16)
    capi.check(capi.lib().sab_test_time_features(R, cand, d, 1, L, time.data_ptr(), tfreq.ptr, mem_base.data_ptr(),
                                                 mem_in.ptr, *([None] * 9), capi.stream_ptr()))
    tf, mi = tfreq.check("tfreq"), mem_in.check("mem_in")
    k = torch.arange(128, device=DEV, dtype=torch.float64)
    a = time.double().view(-1, 1) * torch.exp(-math.log(1e4) * k / 128)
    r = torch.cat([torch.cos(a), torch.sin(a)], 1)
    arg = torch.cat([a, a], 1).abs()
    assert_bound(tf, r, 2.0 ** -8 * r.abs() + 2.0 ** -20 + 2.0 ** -21 * arg, "tfreq")
    half = d // 2
    kk = torch.arange(half, device=DEV, dtype=torch.float64)
    tc = time.double()[::cand].repeat_interleave(L).view(-1, 1)       # the first candidate's time, per text row
    a = tc * torch.exp(-math.log(1e4) * kk / half)
    r = mem_base.double() + torch.cat([torch.cos(a), torch.sin(a)], 1)
    arg = torch.cat([a, a], 1).abs()
    assert_bound(mi, r, 2.0 ** -8 * r.abs() + 2.0 ** -20 + 2.0 ** -21 * arg + 2.0 ** -24 * mem_base.double().abs(),
                 "mem_time")


@gpu
@pytest.mark.parametrize("n_layers,R,d", [(3, 5, 384), (12, 7, 1152)])
def test_build_mod_and_norm_tables_exact(capi, n_layers, R, d):
    """The adaLN tables: mod = table + t0 and fin = final_table + t (fp32 adds), cs = w (1 + scale) and the bf16 shift,
    bit-exact; L B 6 d = 34560 (under one grid stride) and 580608 (not a multiple of the 512 x 256 x 4 stride)."""
    g = gen(n_layers * R)
    tables, t0 = randn(g, n_layers, 6, d), randn(g, R, 6 * d)
    ftable, t = randn(g, 2, d), randn(g, R, d)
    norm_w = 1 + 0.1 * randn(g, 2 * n_layers, d)
    mod, fin = Buf((n_layers, R, 6, d), torch.float32), Buf((R, 2, d), torch.float32)
    cs, shift = Buf((2 * n_layers, R, d), torch.float32), Buf((2 * n_layers, R, d), torch.bfloat16)
    capi.check(capi.lib().sab_test_time_features(R, 1, d, n_layers, 1, None, None, None, None, tables.data_ptr(),
                                                 t0.data_ptr(), ftable.data_ptr(), t.data_ptr(), mod.ptr, fin.ptr,
                                                 norm_w.data_ptr(), cs.ptr, shift.ptr, capi.stream_ptr()))
    m, f, c, s = mod.check("mod"), fin.check("fin"), cs.check("cs"), shift.check("shift")
    r_mod = tables.view(n_layers, 1, 6, d) + t0.view(1, R, 6, d)
    assert torch.equal(m, r_mod), "build_mod: mod"
    assert torch.equal(f, ftable.view(1, 2, d) + t.view(R, 1, d)), "build_mod: fin"
    k = torch.arange(2 * n_layers, device=DEV)
    rows = r_mod[k // 2]                                              # [2L, R, 6, d]
    r0 = (k % 2) * 3
    sh = torch.stack([rows[i, :, r0[i]] for i in range(2 * n_layers)])
    sc = torch.stack([rows[i, :, r0[i] + 1] for i in range(2 * n_layers)])
    assert torch.equal(c, norm_w.view(2 * n_layers, 1, d) * (1 + sc)), "norm_tables: cs"
    assert torch.equal(s.view(torch.int16), sh.bfloat16().view(torch.int16)), "norm_tables: shift"


# ------------------------------------------------------------------------------------------------ RoPE table
@gpu
def test_rope_table_at_max_positions(capi):
    """rope_table at T = max_positions = 10000, theta = 20000, hd = 128, where the fp32 phase error is largest: against
    float64 and against the reference's own fp32 formula (rope.py precompute_freqs_cis: 1 / theta ** (arange(0, hd, 2) /
    hd), torch.outer(t, freqs), cos / sin)."""
    T, hd, theta = 10000, 128, 20000.0
    out = Buf((T, hd // 2, 2), torch.float32)
    capi.check(capi.lib().sab_test_rope_table(T, hd, theta, out.ptr, capi.stream_ptr()))
    o = out.check("rope")
    pos = torch.arange(T, device=DEV, dtype=torch.float64).view(-1, 1)
    inv = theta ** (-torch.arange(0, hd, 2, device=DEV, dtype=torch.float64) / hd)
    a = pos * inv
    tol = (2.0 ** -22 * a.abs() + 2.0 ** -22).unsqueeze(-1)
    r = torch.stack([torch.cos(a), torch.sin(a)], -1)
    assert_bound(o, r, tol.expand_as(r), "rope vs float64")
    freqs = 1.0 / (theta ** (torch.arange(0, hd, 2)[: hd // 2].float() / hd))
    f32 = torch.outer(torch.arange(T), freqs).float()
    r32 = torch.stack([f32.cos(), f32.sin()], -1).to(DEV)
    assert_bound(o, r32, tol.expand_as(r), "rope vs the reference's fp32 formula")


# ------------------------------------------------------------------------------------------------ codec end layers
CODEC_S = [7, 129, 1920 * 3, 1920 * 3 + 5, 128 * 5 + 1]


def check_edges(o, r, tol, what):
    """The first and last 4 samples of every item (the zero-padded taps), reported on their own."""
    for sl, where in ((slice(0, 4), "first"), (slice(-4, None), "last")):
        assert_bound(o[:, sl], r[:, sl], tol[:, sl], f"{what}: {where} 4 samples")


@gpu
@pytest.mark.parametrize("variant", [0, 1, -1])
@pytest.mark.parametrize("C0", [64, 32])
def test_enc_conv0(capi, C0, variant):
    """encoder.block.0 (Conv1d 1 -> C0, k = 7, pad 3, then Snake) in both variants, segment tails (S not a multiple of
    the 128-sample tiles or the hop), per-channel alphas down to 0.05 where the Snake bound is widest."""
    items = 2
    for S in CODEC_S:
        g = gen(S + C0 + variant)
        wav = randn(g, items, S, scale=0.5)
        w, bias = randn(g, C0, 7, scale=0.4), randn(g, C0, scale=0.1)
        alpha = torch.linspace(0.05, 2.0, C0, device=DEV)[torch.randperm(C0, device=DEV, generator=g)]
        x_out, a_out = Buf((items, S, C0), torch.float32), Buf((items, S, C0), torch.bfloat16)
        capi.check(capi.lib().sab_test_codec_end(0, variant, items, S, C0, wav.data_ptr(), w.data_ptr(), bias.data_ptr(),
                                                 alpha.data_ptr(), x_out.ptr, a_out.ptr, None, capi.stream_ptr()))
        x, a = x_out.check("enc.conv0 x_out"), a_out.check("enc.conv0 a_out")
        wp = torch.nn.functional.pad(wav.double(), (3, 3))
        win = wp.unfold(1, 7, 1)                                      # [items, S, 7]: wav[t + k - 3]
        r = win @ w.double().t() + bias.double()
        tol = 2.0 ** -21 * (win.abs() @ w.double().abs().t() + bias.double().abs())
        what = f"enc.conv0 C0={C0} variant={variant} S={S}"
        assert_bound(x, r, tol, what + " x_out")
        check_edges(x, r, tol, what + " x_out")
        al = alpha.double()
        xd = x.double()
        ra = xd + torch.sin(al * xd) ** 2 / (al + 1e-9)
        tola = 2.0 ** -8 * ra.abs() + snake_bound(xd, al)
        assert_bound(a, ra, tola, what + " a_out")
        check_edges(a, ra, tola, what + " a_out")


@gpu
@pytest.mark.parametrize("C,variant", [(64, 1), (96, 1), (128, 1), (64, 0), (96, 0), (128, 0), (160, 0), (96, -1),
                                       (160, -1)])
def test_dec_last(capi, C, variant):
    """The decoder's last conv (C -> 1, k = 7, pad 3) + tanh in the register kernel (C = 64, 96, 128) and the generic one
    (every C, and C = 160 that only it takes), segment tails, the first and last 4 samples of each item."""
    items = 3
    for S in CODEC_S:
        g = gen(S * 3 + C + variant)
        a = bf(randn(g, items, S, C))
        w, bias = randn(g, C, 7, scale=(7 * C) ** -0.5), randn(g, 1, scale=0.2)
        out = Buf((items, S), torch.float32)
        capi.check(capi.lib().sab_test_codec_end(1, variant, items, S, C, a.data_ptr(), w.data_ptr(), bias.data_ptr(),
                                                 None, None, None, out.ptr, capi.stream_ptr()))
        o = out.check("dec.last")
        ap = torch.nn.functional.pad(a.double(), (0, 0, 3, 3))       # [items, S + 6, C]
        win = ap.unfold(1, 7, 1)                                      # [items, S, C, 7]
        pre = (win * w.double()).sum((-1, -2)) + bias.double()
        mag = (win.abs() * w.double().abs()).sum((-1, -2)) + bias.double().abs()
        r = torch.tanh(pre)
        tol = (1 - r * r) * 2.0 ** -24 * 7 * C * mag + 2.0 ** -22
        what = f"dec.last C={C} variant={variant} S={S}"
        assert_bound(o, r, tol, what)
        check_edges(o, r, tol, what)


# ------------------------------------------------------------------------------------------------ T5
@gpu
def test_t5_norm(capi):
    """T5LayerNorm (RMS, eps 1e-6) with rows not a multiple of 8, rows of very different scale and one where eps
    dominates; bf16 and fp32 outputs in one launch; systematic-error check on the bf16 output."""
    rows, d, eps = 301, 768, 1e-6
    g = gen(5)
    x = randn(g, rows, d) * torch.exp(randn(g, rows, 1, scale=2.0))
    x[3] = 1e-4 * randn(g, d)
    w = 1 + 0.2 * randn(g, d)
    ob, of = Buf((rows, d), torch.bfloat16), Buf((rows, d), torch.float32)
    capi.check(capi.lib().sab_test_t5_norm(rows, d, x.data_ptr(), w.data_ptr(), eps, ob.ptr, of.ptr, capi.stream_ptr()))
    b16, f32 = ob.check("t5_norm bf16"), of.check("t5_norm fp32")
    xd = x.double()
    r = xd * torch.rsqrt(xd.pow(2).mean(-1, keepdim=True) + eps) * w.double()
    assert_bound(f32, r, 1e-5 * r.abs(), "t5_norm fp32")
    assert_bound(b16, r, 2.0 ** -8 * r.abs() + 1e-5 * r.abs(), "t5_norm bf16")
    assert torch.equal(b16.view(torch.int16), f32.bfloat16().view(torch.int16)), "bf16 output is not the fp32 one rounded"
    systematic(b16, r, r, 1e-5 * r.abs(), "t5_norm")


@gpu
@pytest.mark.parametrize("L", [1, 13, 32, 33, 100, 171, 172, 512])
def test_t5_attention(capi, L):
    """T5 self-attention with the bucketed relative-position bias table built from t5_relative_buckets(L): one key per
    lane (L <= 32), several (33, 100, 512), the 48 KB dynamic shared-memory threshold (171 | 172) and the ceiling L =
    512; ragged key masks per batch row."""
    from sam_audio_b200.text_encoder import t5_relative_buckets
    B, H = 3, 4
    g = gen(L)
    qkv = bf(randn(g, B * L, 3 * H * 64, scale=0.35))
    rel_w = randn(g, 32, H, scale=2.0)
    bucket = t5_relative_buckets(L).to(DEV)
    mask = torch.zeros(B, L, dtype=torch.uint8, device=DEV)
    for b, n in enumerate((L, max(1, L - 7), max(1, L // 2))):
        mask[b, :n] = 1
    bias, out = Buf((H, 2 * L - 1), torch.float32), Buf((B * L, H * 64), torch.bfloat16)
    capi.check(capi.lib().sab_test_t5_attention(B, L, H, qkv.data_ptr(), rel_w.data_ptr(), bucket.data_ptr(), bias.ptr,
                                                mask.data_ptr(), out.ptr, capi.stream_ptr()))
    tb, o = bias.check("t5 bias table"), out.check("t5 attention")
    assert torch.equal(tb, rel_w[bucket.long()].t()), "t5_bias_table"
    qd = qkv.double().view(B, L, 3, H, 64)
    q, k, v = (qd[:, :, i].transpose(1, 2) for i in range(3))        # [B, H, L, 64]
    i = torch.arange(L, device=DEV)
    delta = i.view(1, -1) - i.view(-1, 1) + L - 1                      # key j - query i, offset
    s = q @ k.transpose(-1, -2) + rel_w.double()[bucket.long()[delta]].permute(2, 0, 1)
    p = torch.softmax(s.masked_fill(~mask.bool()[:, None, None, :], float("-inf")), -1)
    r = (p @ v).transpose(1, 2).reshape(B * L, H * 64)
    mag = (p @ v.abs()).transpose(1, 2).reshape(B * L, H * 64)
    assert_bound(o, r, 2.0 ** -8 * r.abs() + 1e-4 * mag, f"t5_attention L={L}")


@gpu
def test_t5_forward_long_text_vs_float64_transformers(capi):
    """One sab_t5_forward at L = 300 (past the 48 KB attention threshold, where the kernel's shared-memory attribute
    matters) against a float64 copy of the same transformers T5 encoder: ragged texts, valid positions only."""
    import transformers
    from sam_audio_b200.text_encoder import t5_relative_buckets
    cfg = transformers.T5Config(vocab_size=1000, d_model=256, d_kv=64, d_ff=512, num_layers=2, num_heads=4,
                                relative_attention_num_buckets=32, dropout_rate=0.0, feed_forward_proj="relu")
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(0)
        model = transformers.T5EncoderModel(cfg).eval()
    B, L = 2, 300
    gcpu = torch.Generator().manual_seed(1)
    ids = torch.randint(2, cfg.vocab_size, (B, L), generator=gcpu)
    mask = torch.ones(B, L, dtype=torch.long)
    mask[1, 211:] = 0
    ids[1, 211:] = 0
    eng = capi.T5Engine(cfg, 0)
    try:
        eng.load_state_dict(model.state_dict())
        out = torch.empty(B, L, cfg.d_model, device=DEV)
        eng.forward(ids.to(DEV), mask.to(torch.uint8).to(DEV), t5_relative_buckets(L).to(DEV), out)
        torch.cuda.synchronize()
    finally:
        eng.close()
    ref_model = model.double().to(DEV)
    with torch.no_grad():
        ref = ref_model(input_ids=ids.to(DEV), attention_mask=mask.to(DEV))["last_hidden_state"]
    m = mask.to(DEV).bool()
    assert torch.isfinite(out[m]).all()
    assert rel_l2(out[m], ref[m]) <= 2e-2


# ------------------------------------------------------------------------------------------------ host-only rules
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    return _capi.lib()


F = _FAKE
_RMS = dict(M=8, d=1024, x=F, w=F, shift=F, scale=F, mod_ld=0, rows_per_item=8, eps=1e-5, reverse=0, out=F)
_GN = dict(items=1, n=1024, C=64, x=F, gamma=F, beta=F, eps=1e-5, y=F)
_TF = dict(R=4, cand=2, d=256, n_layers=1, L=3, time=F, tfreq=F, mem_base=F, mem_in=F, tables=None, t0=None,
           ftable=None, t=None, mod=None, fin=None, norm_w=None, cs=None, shift=None)
_CF = dict(B=1, cand=1, T=4, d=256, cond=F, cond_clip=F, vproj=F, ln_w=F, ln_b=F, vid_bias=F, vconst=F, gate_v=F,
           emb=F, proj=F, n_anchor=4, adim=128, table=F, ids=F, n_ids=4, align=F, gate_a=F, flags=0)
_CE = dict(which=0, variant=-1, items=1, S=100, C=64, inp=F, w=F, bias=F, alpha=F, x_out=F, a_out=F, wav_out=F)
_AX = dict(items=2, heads=1, Tq=4, Tk=3, cand=1, q=F, k=F + 4096, v=F, mask=None, o=F)
_T5A = dict(B=1, L=8, H=2, qkv=F, rel_w=F, bucket=F, bias=F, mask=F, out=F)


def _call(lib, seam, kw):
    fn = getattr(lib, "sab_test_" + seam)
    rc = fn(*kw.values(), None)
    return None if rc == 0 else lib.sab_last_error().decode()


@pytest.mark.parametrize("seam,base,fields,message", [
    ("rmsnorm_mod", _RMS, dict(d=640), "no instantiation for d=640"),
    ("rmsnorm_mod", _RMS, dict(d=100), "no instantiation for d=100"),
    ("rmsnorm_mod", _RMS, dict(M=0), "M=0 and rows_per_item=8 must be >= 1"),
    ("rmsnorm_mod", _RMS, dict(rows_per_item=0), "rows_per_item=0 must be >= 1"),
    ("rmsnorm_mod", _RMS, dict(mod_ld=6), "mod_ld=6 must be a non-negative multiple of 4"),
    ("rmsnorm_mod", _RMS, dict(reverse=2), "reverse=2 must be 0 or 1"),
    ("rmsnorm_mod", _RMS, dict(shift=F + 8), "16-byte aligned"),
    ("rmsnorm_mod", _RMS, dict(x=None), "null argument"),
    ("group_norm_silu", _GN, dict(C=6), "C=6 must be a positive multiple of 4"),
    ("group_norm_silu", _GN, dict(n=1000), "n_per_item=1000 must be a multiple of C=64"),
    ("group_norm_silu", _GN, dict(items=0), "items=0 outside 1..65535"),
    ("group_norm_silu", _GN, dict(items=70000), "items=70000 outside 1..65535"),
    ("time_features", _TF, dict(R=5), "R=5 must be a positive multiple of cand=2"),
    ("time_features", _TF, dict(d=6), "d=6 must be a positive multiple of 4"),
    ("time_features", _TF, dict(mem_base=None), "mem_in needs mem_base"),
    ("time_features", _TF, dict(time=None), "tfreq / mem_in need time"),
    ("time_features", _TF, dict(mod=F), "mod needs tables, t0, ftable, t and fin"),
    ("time_features", _TF, dict(cs=F), "cs needs mod, norm_w and shift"),
    ("cond_finish", _CF, dict(cond_clip=F + 4096), "cond aliases cond_clip exactly when cand == 1"),
    ("cond_finish", _CF, dict(cand=2), "cond aliases cond_clip exactly when cand == 1"),
    ("cond_finish", _CF, dict(ids=None), "anchor tensors missing"),
    ("cond_finish", _CF, dict(n_ids=0), "anchor tensors missing"),
    ("cond_finish", _CF, dict(flags=4), "unknown flags 4"),
    ("cond_finish", _CF, dict(T=0), "bad shape"),
    ("cond_finish", _CF, dict(n_anchor=0), "n_anchor=0 and anchor_dim=128 must be >= 1"),
    ("codec_end", _CE, dict(which=2), "which=2 must be 0 (enc.conv0) or 1 (dec.last)"),
    ("codec_end", _CE, dict(variant=2), "variant=2 must be -1, 0 or 1"),
    ("codec_end", _CE, dict(S=0), "bad shape"),
    ("codec_end", _CE, dict(C=66), "C0=66 must be a positive multiple of 4"),
    ("codec_end", _CE, dict(C=96, variant=1), "the register kernel needs C0/4 to divide 256 (C0=96)"),
    ("codec_end", _CE, dict(a_out=None), "enc.conv0 needs alpha, x_out and a_out"),
    ("codec_end", _CE, dict(which=1, C=160, variant=1), "the register kernel takes C = 64, 96 or 128 (C=160)"),
    ("codec_end", _CE, dict(which=1, C=192, variant=0), "C=192 needs 57372 B of shared memory"),
    ("codec_end", _CE, dict(which=1, C=63), "C=63 must be even"),
    ("codec_end", _CE, dict(which=1, wav_out=None), "dec.last needs wav_out"),
    ("attention_cross", _AX, dict(k=F), "k == q selects self-attention"),
    ("attention_cross", _AX, dict(cand=3), "items=2 must be a multiple of cand=3"),
    ("attention_cross", _AX, dict(Tk=0), "bad shape"),
    ("attention_cross", _AX, dict(v=F + 2), "16-byte aligned"),
    ("t5_attention", _T5A, dict(L=513), "1 <= L <= 512"),
    ("t5_attention", _T5A, dict(L=0), "1 <= L <= 512"),
    ("t5_attention", _T5A, dict(H=0), "bad shape"),
    ("t5_attention", _T5A, dict(mask=None), "null argument"),
])
def test_simt_seam_rules_rejected(lib, seam, base, fields, message):
    """Host-only: every seam refuses arguments its kernels would mis-handle, with the rule in the message, before any
    CUDA call (so this runs without a GPU)."""
    err = _call(lib, seam, dict(base, **fields))
    assert err is not None and message in err, err


def test_simt_seam_rules_rejected_misc(lib):
    """Host-only: the remaining seams' rules (RoPE table shape, T5 norm outputs)."""
    assert lib.sab_test_rope_table(0, 128, 2e4, F, None) != 0 and b"bad shape (T=0" in lib.sab_last_error()
    assert lib.sab_test_rope_table(10, 127, 2e4, F, None) != 0 and b"hd=127" in lib.sab_last_error()
    assert lib.sab_test_rope_table(10, 128, 1.0, F, None) != 0 and b"theta=1 must be > 1" in lib.sab_last_error()
    assert lib.sab_test_t5_norm(8, 64, F, F, 1e-6, None, None, None) != 0 and b"at least one output" in lib.sab_last_error()
    assert lib.sab_test_t5_norm(0, 64, F, F, 1e-6, F, None, None) != 0 and b"bad shape (rows=0" in lib.sab_last_error()
