"""SAMAudio — H100 drop-in for the reference's ``model.separate()`` path.

Same public surface as the reference class (reference: sam_audio/model/model.py:75-359,
sam_audio/model/base.py:17-62): ``SAMAudio.from_pretrained``, ``.eval()/.to()/.cuda()``,
``.sample_rate``, ``.separate(batch, noise=None, ode_opt=DFLT_ODE_OPT,
reranking_candidates=1, predict_spans=False) -> SeparationResult``, ``.forward`` (one ODE
function evaluation), ``.unbatch``.  All arithmetic of the path runs in
libsamaudio_b200.so (hand-written sm_90a kernels) through the C ABI in
include/samaudio_b200.h; this file only moves pointers and mirrors control flow.
There is no PyTorch / CPU fallback: without the library and an H100 it raises.
"""
from __future__ import annotations

import json
import os
import re
from dataclasses import dataclass
from typing import Any, Dict, List, Optional

import torch
import torch.nn.functional as F

from . import _capi
from .config import SAMAudioConfig
from .processor import Batch
from .text_encoder import SyntheticTextEncoder, T5TextEncoder

DFLT_ODE_OPT = {"method": "midpoint", "options": {"step_size": 2 / 32}}

_SKIP_PREFIXES = re.compile(r"^(text_encoder|visual_ranker|text_ranker|span_predictor|vision_encoder)\.")


@dataclass
class SeparationResult:
    target: List[torch.Tensor]
    residual: List[torch.Tensor]
    noise: torch.Tensor


def fold_weight_norm(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """w = g * v / ||v||  (norm over all dims but 0), for both torch weight-norm spellings
    (``weight_g/weight_v`` and ``parametrizations.weight.original0/1``)."""
    out: Dict[str, torch.Tensor] = {}
    pending: Dict[str, Dict[str, torch.Tensor]] = {}
    for k, v in state_dict.items():
        m = re.match(r"^(?:(.*)\.)?(weight_g|weight_v|parametrizations\.weight\.original[01])$", k)
        if not m:
            out[k] = v
            continue
        kind = "g" if m.group(2) in ("weight_g", "parametrizations.weight.original0") else "v"
        pending.setdefault(m.group(1) or "", {})[kind] = v
    for base, gv in pending.items():
        g, v = gv["g"].float(), gv["v"].float()
        norm = v.flatten(1).norm(dim=1).view(-1, *([1] * (v.dim() - 1)))
        out[f"{base}.weight" if base else "weight"] = g * v / norm
    return out


def _ode_grid(ode_opt: Dict[str, Any]):
    """(n_steps, method) of a fixed-grid `ode_opt`.  The reference forwards **ode_opt to torchdiffeq.odeint
    (model.py:285-290); its fixed-grid solvers are built."""
    method = ode_opt.get("method", "midpoint")
    if method not in _capi.Engine.ODE_METHODS:
        raise NotImplementedError(f"ode method {method!r}: the fixed-grid solvers {sorted(_capi.Engine.ODE_METHODS)} "
                                  "are implemented (adaptive torchdiffeq solvers are not)")
    step = ode_opt.get("options", {}).get("step_size")
    if step is None:
        raise NotImplementedError("fixed-grid solvers need options={'step_size': ...} (torchdiffeq would otherwise "
                                  "take ONE step over [0, 1])")
    n_steps = round(1.0 / float(step))
    if abs(n_steps * float(step) - 1.0) > 1e-6:
        raise NotImplementedError(f"step_size {step} does not divide [0, 1]")
    return n_steps, method


class SAMAudio(torch.nn.Module):
    config_cls = SAMAudioConfig
    revision = None

    def __init__(self, cfg: SAMAudioConfig, text_encoder: Optional[torch.nn.Module] = None,
                 allow_random_text_encoder: bool = False):
        super().__init__()
        cfg.transformer.check_supported()
        self.cfg = cfg
        if text_encoder is None:
            text_encoder = T5TextEncoder(cfg.text_encoder, allow_random_init=allow_random_text_encoder)
        self.text_encoder = text_encoder
        # PE-Core-L14-336 (third party, absent): the wrapper — native frame pre-processing + chunked encode — is built;
        # attach the tower with  model.vision_encoder = PerceptionEncoder(cfg.vision_encoder, model=<CLIP>)
        from .vision_encoder import PerceptionEncoder
        self.vision_encoder = PerceptionEncoder(cfg.vision_encoder)
        # PE-A-Frame span predictor (third party, absent here): attach `span_predictor` + `span_predictor_transform`
        # with the reference's call signatures (model.py:96-102) to enable predict_spans=True.
        self.visual_ranker = None       # third-party scoring models (default config: None): attach any module honouring
        self.text_ranker = None         # the contract in sam_audio_b200/ranking.py; selection follows the reference
        self._engine: Optional[_capi.Engine] = None
        self._state: Optional[Dict[str, torch.Tensor]] = None
        self._plan_limits: Dict[int, Any] = {}          # open stream groups' plan residency (_hold_plan_limits)
        self._device = torch.device("cpu")
        self.register_buffer("_anchor", torch.zeros(1), persistent=False)

    # ------------------------------------------------------------------ loading
    # keyword arguments huggingface_hub.ModelHubMixin.from_pretrained consumes itself (the reference inherits them,
    # base.py:17-45): they go to snapshot_download, never to the constructor
    _HUB_KWARGS = ("force_download", "resume_download", "proxies", "token", "cache_dir", "local_files_only", "revision")

    @classmethod
    def from_pretrained(cls, model_id: str, map_location: str = "cpu", strict: bool = True, **model_kwargs):
        hub = {k: model_kwargs.pop(k) for k in cls._HUB_KWARGS if k in model_kwargs}
        if os.path.isdir(model_id):
            root = model_id
        else:
            from huggingface_hub import snapshot_download
            hub.setdefault("revision", cls.revision)
            hub.pop("resume_download", None)            # accepted for compatibility; deprecated upstream
            root = snapshot_download(repo_id=model_id, **hub)
        with open(os.path.join(root, "config.json")) as f:
            config = json.load(f)
        ctor_kwargs = {}
        for k, v in model_kwargs.items():
            # reference base.py:49-51: keyword arguments override config keys; anything else (and ready-made
            # modules such as text_encoder=...) goes to the constructor
            if k in config and not isinstance(v, torch.nn.Module):
                config[k] = v
            else:
                ctor_kwargs[k] = v
        model = cls(cls.config_cls(**config), **ctor_kwargs)
        sd = torch.load(os.path.join(root, "checkpoint.pt"), weights_only=True, map_location=map_location)
        model.load_state_dict(sd, strict=strict)
        return model

    def load_state_dict(self, state_dict, strict: bool = True):
        """Same tolerance as the reference (model.py:346-359): encoder / ranker / span-predictor keys are
        loaded elsewhere; everything else must match exactly (checked by the engine)."""
        sd = {k: v for k, v in state_dict.items() if not _SKIP_PREFIXES.match(k)}
        self._state = fold_weight_norm(sd)
        self._strict = bool(strict)
        if self._engine is not None:
            return self._push_weights()
        # the engine (and with it the key check) is created on the first .cuda(); until then nothing is known
        return torch.nn.modules.module._IncompatibleKeys([], [])

    def _push_weights(self):
        """strict=True: any unexpected or missing key raises (reference model.py:356-359).  strict=False: unexpected
        keys are skipped, missing ones keep their zero initialisation, and both lists are returned
        (torch's _IncompatibleKeys) — the codec's key names are an assumption (dacvae source is absent), so a real
        checkpoint that deviates is reported key by key instead of failing on the first one."""
        assert self._engine is not None and self._state is not None
        strict = getattr(self, "_strict", True)
        unexpected: List[str] = []
        try:
            for k, v in self._state.items():
                try:
                    self._engine.load_weight(k, v)
                except RuntimeError as exc:
                    if strict or "unexpected weight" not in str(exc):
                        raise
                    unexpected.append(k)
            missing = self._engine.finalize(allow_missing=not strict)
        except RuntimeError as exc:
            hint = ""
            if "audio_codec." in str(exc):
                hint = (" — the audio_codec.* names follow the Descript-DAC layout that `dacvae` derives from; "
                        "load with strict=False to list every unmatched key")
            raise RuntimeError(f"load_state_dict: {exc}{hint}") from exc
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        dev = self._anchor.device
        if dev != self._device:
            self._device = dev
            if self._engine is not None:
                self._engine.close()
                self._engine = None
        return r

    def _ensure_engine(self) -> _capi.Engine:
        if self._engine is None:
            if self._device.type != "cuda":
                raise RuntimeError("sam_audio_b200.SAMAudio runs on an H100 only: call .cuda() first "
                                   "(there is no CPU path)")
            if self._state is None:
                raise RuntimeError("no weights loaded: call load_state_dict()/from_pretrained() first")
            idx = self._device.index if self._device.index is not None else torch.cuda.current_device()
            with torch.cuda.device(idx):
                self._engine = _capi.Engine(self.cfg, idx)
                self._push_weights()
        return self._engine

    # ------------------------------------------------------------------ properties
    @property
    def sample_rate(self) -> int:
        return self.cfg.audio_codec.sample_rate

    def device(self):
        return self._anchor.device

    # ------------------------------------------------------------------ pieces of separate()
    def _pad(self, wavs: torch.Tensor) -> torch.Tensor:
        hop = self.cfg.audio_codec.hop_length
        n = wavs.size(-1)
        if n % hop:
            return F.pad(wavs, (0, hop - n % hop), "reflect")   # codec.py:72-78
        return wavs

    def _get_audio_features(self, audios: torch.Tensor) -> torch.Tensor:
        eng = self._ensure_engine()
        wav = self._pad(audios.float()).squeeze(1).contiguous()
        B, S = wav.shape
        T = S // self.cfg.audio_codec.hop_length
        feats = torch.empty(B, T, 2 * self.cfg.audio_codec.codebook_dim, device=wav.device, dtype=torch.float32)
        with torch.cuda.device(wav.device):
            eng.encode(wav, feats)
        return feats

    def _install_conditioning(self, audio_features, text_features, text_mask, masked_video_features,
                              anchor_ids, anchor_alignment, audio_pad_mask, candidates: int = 1, flags: int = 0):
        """Per-clip tensors; the `candidates` sequences of a clip share them inside the engine
        (reference _repeat_for_reranking, model.py:193-203, without materialising the copies)."""
        eng = self._ensure_engine()
        B, T, _ = audio_features.shape
        dev = audio_features.device
        if text_features is None:                      # reference forward(text_features=None): time-only memory
            flags |= _capi.PREP_NO_TEXT
            L = 1
        else:
            L = text_features.shape[1]
            text_features = text_features.float().contiguous()
        if anchor_ids is None:                         # reference EmbedAnchors returns its input (model.py:57-58)
            flags |= _capi.PREP_NO_ANCHORS
        else:
            anchor_ids = anchor_ids.long().contiguous()
            anchor_alignment = anchor_alignment.long().contiguous()
        if audio_pad_mask is None:
            audio_pad_mask = torch.ones(B, T, dtype=torch.bool, device=dev)
        if text_mask is None:
            text_mask = torch.ones(B, L, dtype=torch.bool, device=dev)
        vid = None if masked_video_features is None else masked_video_features.float().contiguous()
        with torch.cuda.device(dev):
            eng.prepare(B, candidates, T, L, audio_features.float().contiguous(), text_features,
                        text_mask.to(torch.uint8).contiguous(), vid, anchor_ids, anchor_alignment,
                        audio_pad_mask.to(torch.uint8).contiguous(), flags)

    @torch.inference_mode()
    def forward(self, noisy_audio, audio_features, text_features, time, masked_video_features=None,
                text_mask=None, anchor_ids=None, anchor_alignment=None, audio_pad_mask=None):
        """One ODE function evaluation (reference model.py:130-180)."""
        eng = self._ensure_engine()
        # None arguments mean what they mean in the reference: no video term (align.py:41-42), no anchor term
        # (model.py:57-58), time-only memory (model.py:170-172).  separate() never passes None.
        flags = _capi.PREP_NO_VIDEO_TERM if masked_video_features is None else 0
        self._install_conditioning(audio_features, text_features, text_mask, masked_video_features,
                                   anchor_ids, anchor_alignment, audio_pad_mask, flags=flags)
        out = torch.empty_like(noisy_audio, dtype=torch.float32)
        with torch.cuda.device(noisy_audio.device):
            eng.dit_forward(noisy_audio.float().contiguous(), time.float().contiguous(), out)
        return out

    @torch.inference_mode()
    def separate(self, batch: Batch, noise: Optional[torch.Tensor] = None, ode_opt: Dict[str, Any] = DFLT_ODE_OPT,
                 reranking_candidates: int = 1, predict_spans: bool = False, _on_decoded=None) -> SeparationResult:
        """`_on_decoded(i0, i1, wavs)` (private; sam_audio_b200.parallel): called after the waveforms of sequences
        [i0, i1) are enqueued for decoding, so that a collective on them can overlap the next chunk's decode."""
        c = int(reranking_candidates)
        n_steps, method = _ode_grid(ode_opt)
        eng = self._ensure_engine()

        feats = self._get_audio_features(batch.audios)                      # [B, T, 256]
        text_features, text_mask = self.text_encoder(batch.descriptions)
        B, T, C2 = feats.shape
        video = None
        if batch.masked_video is not None:
            if self.vision_encoder is None:
                raise NotImplementedError("visual prompting needs model.vision_encoder (PerceptionEncoder with the "
                                          "PE-Core tower attached; SURVEY §8f-2)")
            video = self.vision_encoder(batch.masked_video).transpose(1, 2)   # raises if no tower is attached
        # reference behaviour (SURVEY App. A.14, model.py:257-268): the forward arguments (anchor tensors included)
        # are bound BEFORE span prediction; predict_spans rebinds batch.anchor_ids/alignment afterwards, so the
        # predicted spans reach the caller's batch but not this call's audio.
        anchor_ids, anchor_alignment, pad_mask = batch.anchor_ids, batch.anchor_alignment, batch.audio_pad_mask
        if predict_spans and getattr(self, "span_predictor", None) is not None and batch.anchors is None:
            batch = self.predict_spans(batch, feats, batch.audio_pad_mask)
        # a batch longer than the model's position table is solved as overlapping windows (sam_audio_b200.windows)
        windowed = T > self.cfg.transformer.max_positions
        if not windowed:
            self._install_conditioning(feats, text_features, text_mask, video, anchor_ids, anchor_alignment, pad_mask,
                                       candidates=c)
        if noise is None:
            noise = torch.randn(B * c, T, C2, device=feats.device, dtype=torch.float32)
        noise = noise.to(device=feats.device, dtype=torch.float32).contiguous()
        hop = self.cfg.audio_codec.hop_length
        wavs = torch.empty(B * c, 2, T * hop, device=feats.device, dtype=torch.float32)
        with torch.cuda.device(feats.device):
            if windowed:
                from .windows import window_layout
                Tw = self.cfg.transformer.max_positions
                latent = self._solve_windows(feats, text_features, text_mask, video, anchor_ids, anchor_alignment,
                                             pad_mask, window_layout([int(n) for n in batch.sizes], Tw), Tw, noise, c,
                                             n_steps, method)
            else:
                latent = torch.empty_like(noise)
                eng.solve(noise, n_steps, latent, method)
            if _on_decoded is None:
                eng.decode(latent, B * c, T, wavs)
            else:                                                           # whole clips (all candidates) per chunk
                step = max(1, int(getattr(self, "decode_chunk_clips", 7))) * c
                for i0 in range(0, B * c, step):
                    i1 = min(B * c, i0 + step)
                    eng.decode(latent[i0:i1], i1 - i0, T, wavs[i0:i1])
                    _on_decoded(i0, i1, wavs)
        self._last_latent = latent                                          # diagnostics (parity tests, bench gate)

        sizes = (batch.sizes * hop).int()                                   # codec.py:91-97
        tgt = self.unbatch(wavs[:, 0].view(B, c, -1), sizes)
        res = self.unbatch(wavs[:, 1].view(B, c, -1), sizes)
        # candidate selection exactly as the reference (model.py:306-330): visual ranker when there is masked video,
        # else text ranker, else candidate 0.  The rankers themselves are third-party modules the caller attaches
        # (sam_audio_b200.ranking documents the contract); the default config has none.
        if c > 1 and batch.masked_video is not None and self.visual_ranker is not None:
            scores = self.visual_ranker(extracted_audio=tgt, videos=batch.masked_video, sample_rate=self.sample_rate)
            idxs = scores.argmax(dim=1)
        elif c > 1 and self.text_ranker is not None:
            input_audio = [audio[:, :size].expand(c, -1) for audio, size in zip(batch.audios, sizes)]
            scores = self.text_ranker(extracted_audio=tgt, input_audio=input_audio, descriptions=batch.descriptions,
                                      sample_rate=self.sample_rate)
            idxs = scores.argmax(dim=1)
        else:
            idxs = torch.zeros(B, dtype=torch.long, device=noise.device)    # model.py:329-330
        idxs = [int(i) for i in idxs]
        return SeparationResult(target=[w[i] for w, i in zip(tgt, idxs)],
                                residual=[w[i] for w, i in zip(res, idxs)], noise=noise)

    def _solve_windows(self, feats, text_features, text_mask, video, anchor_ids, anchor_alignment, pad_mask, wins,
                       Tw: int, noise, c: int, n_steps: int, method: str) -> torch.Tensor:
        """The ODE solve of a batch cut into windows of Tw frames (`wins`, a list of windows.Window; separate() passes
        window_layout(sizes, max_positions)): the windows are solved in groups of bounded size as clips of their own,
        and their latents are cross-faded on the device into latent [B * c, T, 256].  A window's inputs are copies of
        its clip's frames (text, text mask and anchor ids: the clip's own), its noise rows are
        noise[clip * c + k, start:start + Tw], so overlapping windows start from the same noise there.  Every window
        must lie inside [0, T)."""
        from .windows import window_groups, window_ramp, window_rows_budget
        eng = self._ensure_engine()
        B, T, C2 = feats.shape
        dev = feats.device
        noise_bc = noise.view(B, c, T, C2)
        win_lat = torch.empty(len(wins) * c, Tw, C2, device=dev, dtype=torch.float32)   # window-major, candidate-minor
        for i, w in enumerate(wins):
            win_lat[i * c:(i + 1) * c] = noise_bc[w.clip, :, w.start:w.start + Tw]

        def cut(x, time_dim=1):           # [B, T, ...] (or [B, C, T]) -> the group's windows
            if x is None:
                return None
            return torch.stack([x[w.clip].narrow(time_dim - 1, w.start, Tw) for w in grp])

        def per_clip(x):                  # the clip's own row, once per window
            return None if x is None else torch.stack([x[w.clip] for w in grp])
        for w0, w1 in window_groups(len(wins), c, Tw, window_rows_budget()):
            grp = wins[w0:w1]
            self._install_conditioning(cut(feats), per_clip(text_features), per_clip(text_mask), cut(video, 2),
                                       per_clip(anchor_ids), cut(anchor_alignment), cut(pad_mask), candidates=c)
            rows = win_lat[w0 * c:w1 * c]
            eng.solve(rows, n_steps, rows, method)
        seq = torch.tensor([w.clip * c + k for w in wins for k in range(c)], dtype=torch.int32)
        start = torch.tensor([w.start for w in wins for _ in range(c)], dtype=torch.int32)
        flags = torch.tensor([_capi.WIN_FIRST * w.first + _capi.WIN_LAST * w.last for w in wins for _ in range(c)],
                             dtype=torch.uint8)
        latent = torch.empty(B * c, T, C2, device=dev, dtype=torch.float32)
        return _capi.blend_windows(win_lat, seq.to(dev), start.to(dev), flags.to(dev), window_ramp(Tw), latent)

    @torch.inference_mode()
    def resample(self, wav: torch.Tensor, orig_sr: int, new_sr: int) -> torch.Tensor:
        """Band-limited resampling on the GPU (sab_resample; torchaudio's default sinc_interp_hann design):

            x48 = model.resample(x16, 16000, model.sample_rate)     # bring a tensor to the codec's rate ...
            out = model.separate(processor(descriptions=["dog barking"], audios=[x48[None]]).to("cuda"))
            y16 = model.resample(out.target[0], model.sample_rate, 16000)   # ... and the result back

        wav: fp32 [S] or [N, S] (rows are separate signals) on the model's device; one side of the pair must be the
        model's rate, and rates are integers in [8000, 192000] Hz.  Returns [S'] or [N, S'] with S' = ceil(new * S /
        orig) (gcd-reduced), every row in one launch; wav itself when orig_sr == new_sr."""
        from .resample import check_rate, resampled_length
        orig, new = check_rate(orig_sr, "orig_sr"), check_rate(new_sr, "new_sr")
        if self.sample_rate not in (orig, new):
            raise ValueError(f"resampling {orig} -> {new} Hz: one side must be the model's rate ({self.sample_rate} Hz)")
        if not isinstance(wav, torch.Tensor) or wav.dim() not in (1, 2) or wav.shape[-1] < 1:
            raise ValueError(f"resample() takes [S] or [N, S] samples with S >= 1, got "
                             f"{tuple(wav.shape) if isinstance(wav, torch.Tensor) else type(wav).__name__}")
        if wav.dtype != torch.float32 or wav.device != self._device or self._device.type != "cuda":
            raise ValueError(f"resample() takes fp32 samples on the model's CUDA device ({self._device}), got "
                             f"{wav.dtype} on {wav.device}")
        if orig == new:
            return wav
        rows = wav.reshape(-1, wav.shape[-1]).contiguous()
        N, S = rows.shape
        S2 = resampled_length(S, orig, new)
        out = torch.empty(N, S2, device=wav.device, dtype=torch.float32)
        segs = [dict(orig_rate=orig, new_rate=new, in_=rows[i].data_ptr(), in_count=S, length=S,
                     out=out[i].data_ptr(), out_first=0, out_count=S2) for i in range(N)]
        with torch.cuda.device(wav.device):
            self._ensure_engine().resample(segs)
        return out if wav.dim() == 2 else out[0]

    @torch.inference_mode()
    def spread_channels(self, target: torch.Tensor, residual: torch.Tensor, mixture: torch.Tensor):
        """Stereo and surround stems from one mono separation (sab_spread_channels, DESIGN.md section 3): the mono
        target and residual define a time-frequency Wiener mask (STFT of 2048 samples, hop 512, periodic Hann), and the
        mask is applied to every channel of the mixture, so the stems keep its spatial image:

            x48 = model.resample(wav, 44100, model.sample_rate)            # [C, S] channels at the codec's rate
            out = model.separate(processor(descriptions=["piano"], audios=[x48.mean(0, keepdim=True)]).to("cuda"))
            tgt, res = model.spread_channels(out.target[0], out.residual[0], x48)   # [C, S'] each

        target, residual: fp32 [S'] at the model's rate on its CUDA device; mixture: fp32 [C, S], 1 <= C <= 8,
        1 <= S <= S' (zero past S).  Returns (target [C, S'], residual [C, S']) with residual = mixture - target in
        each channel, one fp32 subtraction, all in one launch."""
        from .channels import check_spread_shapes
        C, S, S2 = check_spread_shapes(target, residual, mixture)
        for t in (target, residual, mixture):
            if t.dtype != torch.float32 or t.device != self._device or self._device.type != "cuda":
                raise ValueError(f"spread_channels() takes fp32 samples on the model's CUDA device ({self._device}), "
                                 f"got {t.dtype} on {t.device}")
        t, r, x = target.contiguous(), residual.contiguous(), mixture.contiguous()
        out = torch.empty(2, C, S2, device=t.device, dtype=torch.float32)
        seg = dict(channels=C, target=t.data_ptr(), residual=r.data_ptr(), tr_first=0, tr_count=S2, tr_length=S2,
                   mix=x.data_ptr(), mix_channel_stride=S, mix_first=0, mix_count=S, mix_length=S,
                   out_target=out[0].data_ptr(), out_residual=out[1].data_ptr(), out_channel_stride=S2, out_first=0,
                   out_count=S2)
        with torch.cuda.device(t.device):
            self._ensure_engine().spread_channels([seg])
        return out[0], out[1]

    def _stream_args(self, window_seconds: float, ode_opt: Dict[str, Any], reranking_candidates: int, anchors,
                     masked_video):
        """(W, n_steps, method) of a stream, after the checks stream() and stream_group() share."""
        from .windows import stream_window_frames
        cc = self.cfg.audio_codec
        W = stream_window_frames(window_seconds, cc.sample_rate / cc.hop_length, self.cfg.transformer.max_positions)
        if int(reranking_candidates) != 1:
            raise NotImplementedError("a stream has one candidate: the rankers that choose among candidates score whole "
                                      "clips, which a stream never holds")
        if anchors is not None:
            raise NotImplementedError("a stream takes no anchors: anchor spans are times in a clip, and a stream has no "
                                      "time base for them yet")
        if masked_video is not None:
            raise NotImplementedError("a stream takes no masked video: video frames would need a time base aligned with "
                                      "the stream, which it does not have yet")
        n_steps, method = _ode_grid(ode_opt)
        return W, n_steps, method

    def stream(self, description: str, window_seconds: float = 10.0, seed: int = 0,
               ode_opt: Dict[str, Any] = DFLT_ODE_OPT, reranking_candidates: int = 1, anchors=None,
               masked_video=None, sample_rate: Optional[int] = None, keep_channels: bool = False):
        """Separation of audio that arrives in chunks (sam_audio_b200.stream, DESIGN.md section 3):

            s = model.stream(description="man speaking", sample_rate=16000)
            for chunk in source:          # [S], [1, S] or [C, S] (C <= 8) float samples at sample_rate, any S >= 1
                out = s.push(chunk)       # out.target / out.residual: the samples that became final, at sample_rate
            tail = s.flush()              # the rest; the stream is closed afterwards

        sample_rate: an integer in [8000, 192000] Hz (None: the model's rate).  Channels are averaged.  At another rate
        the stream runs at the model's rate between two resamplers, and its output equals, bit for bit,
        resample(out, model rate, sample_rate) of the model-rate stream pushed resample(channel mean, sample_rate, model
        rate), whatever the chunking.

        keep_channels=True: the outputs are [C, S], the stems of every pushed channel (C from the first push).  The mono
        separation above runs unchanged, and its model-rate target and residual define a Wiener mask that is applied to
        each channel at the model's rate (spread_channels), so the stems keep the input's spatial image and each
        channel's target and residual sum to that channel.  The output equals, bit for bit, resample(spread_channels(T,
        R, x), model rate, sample_rate), with T, R the model-rate stream's output and x the channels at the model's rate
        (resample(x, sample_rate, model rate) row by row), whatever the chunking.  It adds at most 2048 samples at the
        model's rate (42.7 ms) of latency.

        The stream is solved as windows of W = round(window_seconds * 25) latent frames, 8 <= W <= max_positions; the
        default 10 s keeps the DiT on its short-sequence attention (T <= 256).  Text prompts with one candidate only.
        The stream is the one stream of a group of its own (stream_group) that keeps the engine's default plan
        residency."""
        from .stream import StreamGroup
        W, n_steps, method = self._stream_args(window_seconds, ode_opt, reranking_candidates, anchors, masked_video)
        if not isinstance(description, str):
            raise TypeError("a stream separates one source: description must be one string")
        if sample_rate is not None:
            from .resample import check_rate
            check_rate(sample_rate)
        from .stream import check_keep_channels
        check_keep_channels(keep_channels)
        return StreamGroup(self, W, n_steps, method, resident_plans=False).open(description, seed=int(seed),
                                                                                 sample_rate=sample_rate,
                                                                                 keep_channels=keep_channels)

    def stream_group(self, window_seconds: float = 10.0, ode_opt: Dict[str, Any] = DFLT_ODE_OPT,
                     reranking_candidates: int = 1, anchors=None, masked_video=None):
        """Many live streams advanced together (sam_audio_b200.stream, DESIGN.md section 3):

            group = model.stream_group(window_seconds=10.0)
            a = group.open("man speaking", seed=0)      # a stream, with push / flush as from stream()
            c = group.open("rain", sample_rate=16000)    # ... at its own rate and channel count
            d = group.open("piano", keep_channels=True)  # ... with [C, S] stems of every channel (see stream())
            b = group.open("dog barking", seed=7)
            outs = group.push({a: chunk_a, b: chunk_b})  # one tick -> {stream: StreamOutput}
            tails = group.flush([a, b])                  # ends and closes them (a.flush() alone works too)
            group.close()                                # flushes what is still open; also on leaving a `with` block

        Every stream of a group has the same W and ODE grid; prompts and seeds are per stream, and streams may open and
        close at any tick.  A tick solves every window that becomes ready in it, from all its streams, in one batched
        solve, and each stream's output is bit-identical to what stream() returns for the same pushes, whatever the other
        streams do, as long as every prompt of the group has at most 8 tokens (a longer one moves the whole group to the
        unfused cross-attention, whose bits depend on the padded text length).  While the group is open the engine keeps
        one DiT plan per bucket of window counts it has used resident (and the codec plans of those buckets), so ticks
        of varying size do not re-plan; close() restores the default residency, and so does collecting a group dropped
        without close().  A flush tick reuses the buckets of earlier ticks, so ending many streams at once plans no
        larger DiT bucket beside them.

        Offline jobs take the ticks' filler slots (the spare slots of each bucket, otherwise repeated live items):

            job = group.submit(wav, "dog barking", seed=3, sample_rate=16000)   # a whole recording, [S] or [C, S]
                                                                                # (keep_channels as for open())
            group.drain([job])                   # ticks of jobs only, at buckets the group uses; close() drains too
            out = job.result()                   # == model.stream(...) with wav pushed once and flushed, bit for bit

        A job is cut into codec tiles of the steady slice lengths, so in push ticks it adds no planned call, changes no
        call's item count and builds no plan; live streams keep their bits.  The exception is a job prompt longer than
        every prompt of the group: like open(), it raises the group's text length, and the next tick re-plans every
        bucket at it.  submit() copies the recording.  Jobs run first in, first out; job.cancel()
        frees one, and a group collected without close() cancels its jobs."""
        from .stream import StreamGroup
        W, n_steps, method = self._stream_args(window_seconds, ode_opt, reranking_candidates, anchors, masked_video)
        return StreamGroup(self, W, n_steps, method, resident_plans=True)

    def _hold_plan_limits(self, holder, limits) -> None:
        """Engine plan residency: the largest (DiT plans, codec plans per direction) any open stream group holds, the
        engine's defaults when none does.  `holder` is a group's key object; limits=None releases its hold."""
        if limits is None:
            self._plan_limits.pop(id(holder), None)
        else:
            self._plan_limits[id(holder)] = limits
        if self._engine is None:
            return
        held = [_capi.Engine.DEFAULT_PLAN_LIMITS] + list(self._plan_limits.values())
        self._engine.set_plan_limits(max(h[0] for h in held), max(h[1] for h in held))

    def predict_spans(self, batch: Batch, audio_features: torch.Tensor, audio_pad_mask: torch.Tensor) -> Batch:
        """Reference model.py:231-245: frame-level span predictor on the first 128 latent channels -> "+" anchors ->
        ``batch.process_anchors`` (mutates the caller's batch).  At the pinned reference commit the conditioning
        has already been built from the old anchors, so the audio does not change (SURVEY App. A.14)."""
        inputs = self.span_predictor_transform(text=batch.descriptions).to(audio_features.device)
        output = self.span_predictor(input_features=audio_features[:, :, :128], padding_mask=audio_pad_mask,
                                     return_spans=True, **inputs)
        anchors = [[["+"] + list(a) for a in clip] for clip in output.spans]
        batch.process_anchors(anchors)
        return batch

    def unbatch(self, wavs: torch.Tensor, sizes: torch.Tensor, time_dim: int = -1):
        return [row.narrow(dim=time_dim, start=0, length=int(n)) for row, n in zip(wavs, sizes)]

    # ------------------------------------------------------------------ introspection
    def launch_count(self, reset: bool = False) -> int:
        return self._ensure_engine().launch_count(reset)


def build_synthetic_model(name: str = "sam-audio-tiny", seed: int = 0, text: str = "synthetic",
                          device: str = "cuda", weights_device: str = "cpu") -> SAMAudio:
    """Random-init model of a stand-in shape (no checkpoints in the sandbox)."""
    from .config import stand_in_config
    from .synthetic import make_state_dict
    cfg = stand_in_config(name)
    te = SyntheticTextEncoder(cfg.text_encoder.dim) if text == "synthetic" else \
        T5TextEncoder(cfg.text_encoder, allow_random_init=True)
    m = SAMAudio(cfg, text_encoder=te)
    m.load_state_dict(make_state_dict(cfg, seed=seed, device=weights_device))
    return m.eval().to(device)
