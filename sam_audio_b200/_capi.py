"""ctypes binding of libsamaudio_b200.so (include/samaudio_b200.h).

PyTorch is used only as the owner of device memory and streams: every call
passes raw ``data_ptr()`` values and the current CUDA stream.  There is no
fallback: a missing library or a missing GPU raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

_LIB_NAME = "libsamaudio_b200.so"
_lib: Optional[ctypes.CDLL] = None


class SabConfig(ctypes.Structure):
    _fields_ = [
        ("dim", ctypes.c_int32), ("n_heads", ctypes.c_int32), ("n_layers", ctypes.c_int32),
        ("ffn_hidden", ctypes.c_int32), ("out_channels", ctypes.c_int32), ("in_channels", ctypes.c_int32),
        ("text_dim", ctypes.c_int32), ("vision_dim", ctypes.c_int32), ("n_anchor_tokens", ctypes.c_int32),
        ("anchor_dim", ctypes.c_int32), ("max_positions", ctypes.c_int32),
        ("rope_theta", ctypes.c_float), ("norm_eps", ctypes.c_float),
        ("codec_encoder_dim", ctypes.c_int32), ("codec_latent_dim", ctypes.c_int32),
        ("codec_decoder_dim", ctypes.c_int32), ("codec_codebook_dim", ctypes.c_int32),
        ("codec_n_rates", ctypes.c_int32),
        ("codec_encoder_rates", ctypes.c_int32 * 8), ("codec_decoder_rates", ctypes.c_int32 * 8),
    ]


class SabT5Config(ctypes.Structure):
    _fields_ = [("vocab_size", ctypes.c_int32), ("d_model", ctypes.c_int32), ("d_kv", ctypes.c_int32),
                ("d_ff", ctypes.c_int32), ("n_layers", ctypes.c_int32), ("n_heads", ctypes.c_int32),
                ("n_buckets", ctypes.c_int32), ("eps", ctypes.c_float)]


class SabTestGemmRun(ctypes.Structure):
    _fields_ = [("row_shift", ctypes.c_int32), ("a_col", ctypes.c_int32), ("nkb", ctypes.c_int32)]


class SabTestGemmDesc(ctypes.Structure):
    """Mirror of sab_test_gemm_desc (include/samaudio_b200.h); pointers are device addresses as ints."""
    _i32, _i64, _f32, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_float, ctypes.c_void_p
    _fields_ = [
        ("struct_bytes", _i32),
        ("mode", _i32), ("bn", _i32), ("bk", _i32), ("cg", _i32), ("b2b", _i32),
        ("a", _vp), ("a_cols", _i64), ("a_rows", _i64), ("a_items", _i64), ("a_row_pitch", _i64), ("a_item_pitch", _i64),
        ("b", _vp), ("n", _i32), ("w1", _vp),
        ("n_runs", _i32 * 2), ("runs", (SabTestGemmRun * 8) * 2), ("n_period", _i32), ("n_switch", _i32),
        ("grid_ctas", _i32), ("group_m", _i32), ("reverse_m", _i32),
        ("bias", _vp), ("bias_mod", _i32),
        ("gate", _vp), ("gate_ld", _i32), ("gate_div", _i32),
        ("alpha", _f32), ("relu", _i32),
        ("res", _vp), ("res_ld", _i64),
        ("out_f32", _vp), ("out_f32_ld", _i64),
        ("out_bf16", _vp), ("out_bf16_ld", _i64),
        ("out_act", _vp), ("out_act_ld", _i64), ("snake_alpha", _vp),
        ("colscale", _vp), ("colscale_ld", _i64),
        ("out_scaled", _vp), ("out_scaled_ld", _i64),
        ("ssq_out", _vp), ("ssq_ld", _i32),
        ("ssq_in", _vp), ("ssq_n", _i32), ("ssq_inv_dim", _f32),
        ("ibias", _vp), ("ibias_ld", _i64), ("ibias_div", _i32),
        ("b2b_bias", _vp), ("b2b_alpha", _vp),
        ("qnorm_w", _vp), ("knorm_w", _vp),
        ("n_q_end", _i32), ("n_k_end", _i32), ("qkv_period", _i32), ("norm_w_stride", _i32),
        ("rope", _vp), ("rope_T", _i32), ("use_rope", _i32), ("eps", _f32),
        ("xa_kv", _vp), ("xa_kv_ld", _i64), ("xa_v_col0", _i32), ("xa_Tk", _i32), ("xa_T", _i32),
        ("xa_mask", _vp), ("xa_scale_log2", _f32),
        ("b_clip_rows", _i32), ("b_clip_div", _i32), ("b_cols", _i64), ("b_ld", _i64),
        ("xa_p", _vp), ("xa_p_ld", _i64),
    ]

    def __init__(self, **kw):
        super().__init__()
        self.struct_bytes = ctypes.sizeof(SabTestGemmDesc)
        self.alpha, self.gate_div, self.ibias_div, self.eps = 1.0, 1, 1, 1e-5   # the planner's defaults
        for k, v in kw.items():
            setattr(self, k, v)


class SabResampleSeg(ctypes.Structure):
    """Mirror of sab_resample_seg (include/samaudio_b200.h); pointers are device addresses as ints."""
    _i32, _i64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p
    _fields_ = [("struct_bytes", _i32), ("orig_rate", _i32), ("new_rate", _i32), ("channels", _i32),
                ("in_", _vp), ("in_channel_stride", _i64), ("in_first", _i64), ("in_count", _i64),
                ("length", _i64),
                ("out", _vp), ("out_first", _i64), ("out_count", _i64)]

    def __init__(self, **kw):
        super().__init__()
        self.struct_bytes = ctypes.sizeof(SabResampleSeg)
        self.channels, self.length = 1, -1
        for k, v in kw.items():
            setattr(self, k, v)


class SabSpreadSeg(ctypes.Structure):
    """Mirror of sab_spread_seg (include/samaudio_b200.h); pointers are device addresses as ints."""
    _i32, _i64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p
    _fields_ = [("struct_bytes", _i32), ("channels", _i32),
                ("target", _vp), ("residual", _vp), ("tr_first", _i64), ("tr_count", _i64), ("tr_length", _i64),
                ("mix", _vp), ("mix_channel_stride", _i64), ("mix_first", _i64), ("mix_count", _i64),
                ("mix_length", _i64),
                ("out_target", _vp), ("out_residual", _vp), ("out_channel_stride", _i64), ("out_first", _i64),
                ("out_count", _i64)]

    def __init__(self, **kw):
        super().__init__()
        self.struct_bytes = ctypes.sizeof(SabSpreadSeg)
        self.channels, self.tr_length, self.mix_length = 1, -1, -1
        for k, v in kw.items():
            setattr(self, k, v)


EXPORTS = [
    "sab_last_error", "sab_version", "sab_create", "sab_destroy", "sab_load_weight", "sab_finalize_weights",
    "sab_encode", "sab_prepare", "sab_dit_forward", "sab_solve", "sab_decode", "sab_launch_count",
    "sab_workspace_bytes", "sab_set_plan_limits", "sab_plan_stats", "sab_profile", "sab_profile_report", "sab_test_gemm", "sab_test_gemm_ex", "sab_test_xattn_fold", "sab_test_attention", "sab_test_attention_tc2", "sab_test_attention_stream", "sab_codec_tiling", "sab_preprocess_frames", "sab_blend_windows", "sab_test_aa_taps", "sab_test_solver_grid",
    "sab_resample", "sab_resample_taps", "sab_spread_channels",
    "sab_test_rmsnorm_mod", "sab_test_group_norm_silu", "sab_test_time_features", "sab_test_cond_finish",
    "sab_test_rope_table", "sab_test_codec_end", "sab_test_attention_cross", "sab_test_t5_norm", "sab_test_t5_attention",
    "sab_t5_create", "sab_t5_destroy", "sab_t5_load_weight", "sab_t5_finalize", "sab_t5_forward", "sab_t5_launch_count",
]


def library_path() -> str:
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), _LIB_NAME)


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        path = library_path()
        if not os.path.exists(path):
            raise RuntimeError(
                f"{_LIB_NAME} not built ({path}); run `python -c 'import __graft_entry__ as g; g.build()'`. "
                "The H100 separation path has no CPU/PyTorch fallback.")
        L = ctypes.CDLL(path)
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
        L.sab_last_error.restype = ctypes.c_char_p
        L.sab_create.argtypes = [ctypes.POINTER(SabConfig), i32, ctypes.POINTER(vp)]
        L.sab_destroy.argtypes = [vp]
        L.sab_load_weight.argtypes = [vp, ctypes.c_char_p, vp, ctypes.POINTER(i64), i32, i32, vp]
        L.sab_finalize_weights.argtypes = [vp, i32, ctypes.c_char_p, i64, vp]
        L.sab_encode.argtypes = [vp, vp, i32, i64, vp, vp]
        L.sab_prepare.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp, vp, vp, i32, vp, vp, i32, vp]
        L.sab_dit_forward.argtypes = [vp, vp, vp, vp, vp]
        L.sab_solve.argtypes = [vp, vp, i32, i32, vp, vp]
        L.sab_decode.argtypes = [vp, vp, i32, i32, vp, vp]
        L.sab_launch_count.argtypes = [vp, i32]
        L.sab_launch_count.restype = i64
        L.sab_workspace_bytes.argtypes = [vp]
        L.sab_workspace_bytes.restype = i64
        L.sab_set_plan_limits.argtypes = [vp, i32, i32]
        L.sab_plan_stats.argtypes = [vp, ctypes.POINTER(i64), ctypes.POINTER(i64), ctypes.POINTER(i64),
                                     ctypes.POINTER(i32), ctypes.POINTER(i32)]
        L.sab_profile.argtypes = [vp, i32, vp]
        L.sab_profile_report.argtypes = [vp, ctypes.c_char_p, i64, vp]
        L.sab_test_gemm.argtypes = [i32, i32, i32, vp, vp, vp, i32, i32, i32, vp]
        L.sab_test_gemm_ex.argtypes = [ctypes.POINTER(SabTestGemmDesc), vp]
        L.sab_test_xattn_fold.argtypes = [i32, i32, i32, i32, vp, vp, i64, i64, i32, vp, i32, i64, vp]
        L.sab_test_attention.argtypes = [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
        L.sab_test_attention_tc2.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp, ctypes.c_float, i32, vp]
        L.sab_test_attention_stream.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp, ctypes.c_float, i32, vp]
        L.sab_codec_tiling.argtypes = [vp, i32, i32, ctypes.POINTER(i32), ctypes.POINTER(i32)]
        L.sab_preprocess_frames.argtypes = [vp, i32, i32, i32, i32, vp, vp, vp]
        L.sab_blend_windows.argtypes = [vp, i32, i32, vp, vp, vp, i32, vp, i32, i32, vp]
        L.sab_test_aa_taps.argtypes = [i32, i32, i32, vp, vp, vp, vp]
        L.sab_test_solver_grid.argtypes = [i32, i32, i32, vp, vp]
        L.sab_resample.argtypes = [vp, ctypes.POINTER(SabResampleSeg), i32, vp]
        L.sab_resample_taps.argtypes = [i32, i32, i64, ctypes.POINTER(i32), vp, vp]
        L.sab_spread_channels.argtypes = [vp, ctypes.POINTER(SabSpreadSeg), i32, vp]
        f32 = ctypes.c_float
        L.sab_test_rmsnorm_mod.argtypes = [i32, i32, vp, vp, vp, vp, i64, i32, f32, i32, vp, vp]
        L.sab_test_group_norm_silu.argtypes = [i32, i64, i32, vp, vp, vp, f32, vp, vp]
        L.sab_test_time_features.argtypes = [i32, i32, i32, i32, i32] + [vp] * 14
        L.sab_test_cond_finish.argtypes = [i32, i32, i32, i32] + [vp] * 10 + [i32, i32, vp, vp, i32, vp, vp, i32, vp]
        L.sab_test_rope_table.argtypes = [i32, i32, f32, vp, vp]
        L.sab_test_codec_end.argtypes = [i32, i32, i32, i64, i32, vp, vp, vp, vp, vp, vp, vp, vp]
        L.sab_test_attention_cross.argtypes = [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp]
        L.sab_test_t5_norm.argtypes = [i64, i32, vp, vp, f32, vp, vp, vp]
        L.sab_test_t5_attention.argtypes = [i32, i32, i32, vp, vp, vp, vp, vp, vp, vp]
        L.sab_t5_create.argtypes = [ctypes.POINTER(SabT5Config), i32, ctypes.POINTER(vp)]
        L.sab_t5_destroy.argtypes = [vp]
        L.sab_t5_load_weight.argtypes = [vp, ctypes.c_char_p, vp, ctypes.POINTER(i64), i32, i32, vp]
        L.sab_t5_finalize.argtypes = [vp, vp]
        L.sab_t5_forward.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp]
        L.sab_t5_launch_count.argtypes = [vp, i32]
        L.sab_t5_launch_count.restype = i64
        _lib = L
    return _lib


PREP_NO_VIDEO_TERM, PREP_NO_ANCHORS, PREP_NO_TEXT = 1, 2, 4   # include/samaudio_b200.h SAB_PREP_*


def check(rc: int) -> None:
    if rc != 0:
        raise RuntimeError("samaudio_b200: " + lib().sab_last_error().decode("utf-8", "replace"))


def stream_ptr() -> int:
    return torch.cuda.current_stream().cuda_stream


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def make_config(cfg) -> SabConfig:
    """cfg: sam_audio_b200.config.SAMAudioConfig"""
    tc, cc = cfg.transformer, cfg.audio_codec
    c = SabConfig()
    c.dim, c.n_heads, c.n_layers, c.ffn_hidden = tc.dim, tc.n_heads, tc.n_layers, tc.ffn_hidden
    c.out_channels, c.in_channels = tc.out_channels, cfg.in_channels
    c.text_dim, c.vision_dim = cfg.text_encoder.dim, cfg.vision_encoder.dim
    c.n_anchor_tokens, c.anchor_dim = cfg.num_anchors + 1, cfg.anchor_embedding_dim
    c.max_positions, c.rope_theta, c.norm_eps = tc.max_positions, tc.rope_theta, tc.norm_eps
    c.codec_encoder_dim, c.codec_latent_dim = cc.encoder_dim, cc.latent_dim
    c.codec_decoder_dim, c.codec_codebook_dim = cc.decoder_dim, cc.codebook_dim
    c.codec_n_rates = len(cc.encoder_rates)
    assert len(cc.decoder_rates) == len(cc.encoder_rates) <= 8
    for i, r in enumerate(cc.encoder_rates):
        c.codec_encoder_rates[i] = r
    for i, r in enumerate(cc.decoder_rates):
        c.codec_decoder_rates[i] = r
    return c


def preprocess_frames(frames: torch.Tensor, out_size: int) -> torch.Tensor:
    """uint8 [N, 3, H, W] (cuda) -> fp32 [N, 3, S, S]: antialiased bicubic resize, uint8 rounding, (x/255 - .5)/.5."""
    assert frames.is_cuda and frames.dtype == torch.uint8 and frames.dim() == 4 and frames.shape[1] == 3
    frames = frames.contiguous()
    n, _, h, w = frames.shape
    out = torch.empty(n, 3, out_size, out_size, device=frames.device, dtype=torch.float32)
    ws = torch.empty(n, 3, h, out_size, device=frames.device, dtype=torch.float32)
    with torch.cuda.device(frames.device):
        check(lib().sab_preprocess_frames(frames.data_ptr(), n, h, w, out_size, ws.data_ptr(), out.data_ptr(), stream_ptr()))
    return out


WIN_FIRST, WIN_LAST = 1, 2   # include/samaudio_b200.h SAB_WIN_*


def blend_windows(win_latent: torch.Tensor, seq: torch.Tensor, start: torch.Tensor, flags: torch.Tensor, ramp: int,
                  out: torch.Tensor) -> torch.Tensor:
    """win_latent [n_win, Tw, 256] fp32 -> out [Bc, T, 256]: the cross-fade of sab_blend_windows (all tensors on one
    device; seq / start int32, flags uint8 = WIN_FIRST | WIN_LAST, one entry per window)."""
    n_win, Tw, C = win_latent.shape
    Bc, T, C2 = out.shape
    assert C == C2 == 256 and win_latent.dtype == out.dtype == torch.float32
    assert win_latent.is_contiguous() and out.is_contiguous()
    assert seq.dtype == start.dtype == torch.int32 and flags.dtype == torch.uint8
    assert seq.shape == start.shape == flags.shape == (n_win,)
    seq, start, flags = seq.contiguous(), start.contiguous(), flags.contiguous()
    with torch.cuda.device(out.device):
        check(lib().sab_blend_windows(win_latent.data_ptr(), n_win, Tw, seq.data_ptr(), start.data_ptr(),
                                      flags.data_ptr(), int(ramp), out.data_ptr(), Bc, T, stream_ptr()))
    return out


def resample_taps(orig_rate: int, new_rate: int):
    """The table sab_resample uses for a rate pair (host only): (K, lo [n] int32, w [n, K] fp32) as numpy arrays."""
    import math

    import numpy as np
    n = int(new_rate) // math.gcd(int(orig_rate), int(new_rate))
    K = ctypes.c_int()
    check(lib().sab_resample_taps(int(orig_rate), int(new_rate), 0, ctypes.byref(K), None, None))
    lo = np.zeros(n, np.int32)
    w = np.zeros((n, K.value), np.float32)
    check(lib().sab_resample_taps(int(orig_rate), int(new_rate), w.size, ctypes.byref(K), lo.ctypes.data, w.ctypes.data))
    return K.value, lo, w


def resample_segments(segs) -> ctypes.Array:
    """A list of SabResampleSeg (or of dicts of its fields) as the C array sab_resample takes."""
    arr = (SabResampleSeg * max(1, len(segs)))()
    for i, s in enumerate(segs):
        arr[i] = s if isinstance(s, SabResampleSeg) else SabResampleSeg(**s)
    return arr


def spread_segments(segs) -> ctypes.Array:
    """A list of SabSpreadSeg (or of dicts of its fields) as the C array sab_spread_channels takes."""
    arr = (SabSpreadSeg * max(1, len(segs)))()
    for i, s in enumerate(segs):
        arr[i] = s if isinstance(s, SabSpreadSeg) else SabSpreadSeg(**s)
    return arr


class Engine:
    """Owns one sab_engine handle."""

    def __init__(self, cfg, device: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("samaudio_b200: CUDA device required (no CPU fallback)")
        self._h = ctypes.c_void_p()
        self._cfg = make_config(cfg)
        self.device = device
        check(lib().sab_create(ctypes.byref(self._cfg), device, ctypes.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().sab_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_weight(self, name: str, t: torch.Tensor):
        t = t.detach().to(torch.float32).contiguous()
        shape = (ctypes.c_int64 * max(t.dim(), 1))(*(t.shape if t.dim() else (1,)))
        check(lib().sab_load_weight(self._h, name.encode(), t.data_ptr(), shape, max(t.dim(), 1),
                                    1 if t.is_cuda else 0, stream_ptr()))

    def finalize(self, allow_missing: bool = False):
        """Returns the list of missing keys (empty unless allow_missing)."""
        import ctypes as C
        buf = C.create_string_buffer(1 << 16)
        check(lib().sab_finalize_weights(self._h, 1 if allow_missing else 0, buf, len(buf), stream_ptr()))
        return [k for k in buf.value.decode().split("\n") if k]

    def encode(self, wav: torch.Tensor, features: torch.Tensor):
        B, S = wav.shape
        check(lib().sab_encode(self._h, wav.data_ptr(), B, S, features.data_ptr(), stream_ptr()))

    def prepare(self, B, candidates, T, L, features, text, text_mask, video, anchor_ids, anchor_alignment, pad_mask,
                flags=0):
        check(lib().sab_prepare(self._h, B, candidates, T, L, features.data_ptr(), ptr(text), text_mask.data_ptr(),
                                ptr(video), ptr(anchor_ids), 0 if anchor_ids is None else anchor_ids.shape[1],
                                ptr(anchor_alignment), pad_mask.data_ptr(), flags, stream_ptr()))

    def dit_forward(self, noisy, time, out):
        check(lib().sab_dit_forward(self._h, noisy.data_ptr(), time.data_ptr(), out.data_ptr(), stream_ptr()))

    ODE_METHODS = {"midpoint": 0, "euler": 1, "rk4": 2}    # include/samaudio_b200.h SAB_ODE_*

    def solve(self, noise, n_steps, out, method: str = "midpoint"):
        check(lib().sab_solve(self._h, noise.data_ptr(), n_steps, self.ODE_METHODS[method], out.data_ptr(), stream_ptr()))

    def decode(self, latent, Bc, T, wav):
        check(lib().sab_decode(self._h, latent.data_ptr(), Bc, T, wav.data_ptr(), stream_ptr()))

    def launch_count(self, reset=False) -> int:
        return int(lib().sab_launch_count(self._h, 1 if reset else 0))

    def profile(self, enable: bool):
        check(lib().sab_profile(self._h, 1 if enable else 0, stream_ptr()))

    def profile_report(self) -> dict:
        import json
        buf = ctypes.create_string_buffer(1 << 16)
        check(lib().sab_profile_report(self._h, buf, len(buf), stream_ptr()))
        return json.loads(buf.value.decode())

    def codec_tiling(self, decoder: bool, T: int):
        """(halo, tile length) in latent frames for a clip of T frames; tile length 0 = the clip runs whole."""
        halo, tile = ctypes.c_int(), ctypes.c_int()
        check(lib().sab_codec_tiling(self._h, 1 if decoder else 0, T, ctypes.byref(halo), ctypes.byref(tile)))
        return halo.value, tile.value

    def workspace_bytes(self) -> int:
        return int(lib().sab_workspace_bytes(self._h))

    def resample(self, segs) -> None:
        """One sab_resample launch over `segs` (SabResampleSeg or dicts of its fields) on the current stream."""
        if segs:
            check(lib().sab_resample(self._h, resample_segments(segs), len(segs), stream_ptr()))

    def spread_channels(self, segs) -> None:
        """One sab_spread_channels launch over `segs` (SabSpreadSeg or dicts of its fields) on the current stream."""
        if segs:
            check(lib().sab_spread_channels(self._h, spread_segments(segs), len(segs), stream_ptr()))

    DEFAULT_PLAN_LIMITS = (1, 3)    # include/samaudio_b200.h sab_set_plan_limits

    def set_plan_limits(self, dit_plans: int, codec_plans_per_direction: int):
        check(lib().sab_set_plan_limits(self._h, int(dit_plans), int(codec_plans_per_direction)))

    def plan_stats(self) -> dict:
        """Plans built and solve graphs captured since the engine was created, and the plans resident now."""
        b, g, cb = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
        dr, cr = ctypes.c_int(), ctypes.c_int()
        check(lib().sab_plan_stats(self._h, ctypes.byref(b), ctypes.byref(g), ctypes.byref(cb), ctypes.byref(dr),
                                   ctypes.byref(cr)))
        return {"dit_plan_builds": b.value, "graph_captures": g.value, "codec_plan_builds": cb.value,
                "dit_plans_resident": dr.value, "codec_plans_resident": cr.value}


class T5Engine:
    """Owns one sab_t5 handle (native T5 text encoder)."""

    def __init__(self, hf_config, device: int = 0):
        if not torch.cuda.is_available():
            raise RuntimeError("samaudio_b200: CUDA device required (no CPU fallback)")
        c = SabT5Config()
        c.vocab_size, c.d_model, c.d_kv, c.d_ff = hf_config.vocab_size, hf_config.d_model, hf_config.d_kv, hf_config.d_ff
        c.n_layers, c.n_heads = hf_config.num_layers, hf_config.num_heads
        c.n_buckets, c.eps = hf_config.relative_attention_num_buckets, hf_config.layer_norm_epsilon
        self._cfg = c
        self._h = ctypes.c_void_p()
        check(lib().sab_t5_create(ctypes.byref(c), device, ctypes.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().sab_t5_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_state_dict(self, sd):
        for k, v in sd.items():
            t = v.detach().to(torch.float32).contiguous()
            shape = (ctypes.c_int64 * t.dim())(*t.shape)
            check(lib().sab_t5_load_weight(self._h, k.encode(), t.data_ptr(), shape, t.dim(), 1 if t.is_cuda else 0,
                                           stream_ptr()))
        check(lib().sab_t5_finalize(self._h, stream_ptr()))

    def forward(self, ids, mask_u8, rel_bucket, out):
        B, L = ids.shape
        check(lib().sab_t5_forward(self._h, ids.data_ptr(), mask_u8.data_ptr(), rel_bucket.data_ptr(), B, L,
                                   out.data_ptr(), stream_ptr()))

    def launch_count(self, reset=False) -> int:
        return int(lib().sab_t5_launch_count(self._h, 1 if reset else 0))
