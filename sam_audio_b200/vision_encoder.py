"""PerceptionEncoder — host mirror of the reference's visual-prompting encoder wrapper
(reference: sam_audio/model/vision_encoder.py:16-113).

What is built natively: the frame pre-processing (`get_transform`: antialiased bicubic resize to image_size^2 on uint8
frames, /255, Normalize(.5,.5)) as sm_90a kernels behind `sab_preprocess_frames`, and the control flow of
`VisionEncoder.forward` (per-video transform, chunks of `batch_size` frames, zero pad_sequence).  What is NOT here: the
PE-Core-L14-336 CLIP tower itself (third-party `perception-models`, source and weights absent — SURVEY §8f-2): pass it as
`model` (anything with `encode_image(x, normalize=...)`); without one, encoding raises.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from . import _capi
from .config import PerceptionEncoderConfig


class PerceptionEncoder(torch.nn.Module):
    def __init__(self, cfg: Optional[PerceptionEncoderConfig] = None, model: Optional[torch.nn.Module] = None):
        super().__init__()
        cfg = cfg or PerceptionEncoderConfig()
        if cfg.interpolation_mode.upper() != "BICUBIC":
            raise NotImplementedError(f"interpolation_mode {cfg.interpolation_mode!r}: the H100 kernel implements the "
                                      "reference's shipped BICUBIC (antialiased) resize")
        self.batch_size = cfg.batch_size
        self.dim = cfg.dim
        self.normalize_feature = cfg.normalize_feature
        self.image_size = cfg.image_size
        self.name = cfg.name
        self.model = model

    def transform(self, video: torch.Tensor) -> torch.Tensor:
        """[T, 3, H, W] uint8 -> [T, 3, S, S] float32 on the video's (cuda) device — vision_encoder.py:91-113."""
        if video.dtype != torch.uint8:
            raise NotImplementedError("the reference pipeline feeds uint8 frames (torchcodec / mask_videos); the H100 "
                                      "resize kernel reproduces torchvision's uint8 rounding")
        if not video.is_cuda:
            raise RuntimeError("PerceptionEncoder.transform runs on an H100 only: move the frames to cuda (no CPU path)")
        return _capi.preprocess_frames(video, self.image_size)

    def encode(self, x: torch.Tensor) -> torch.Tensor:
        if self.model is None:
            raise NotImplementedError(f"the {self.name} vision tower is third-party (perception-models) and absent here: "
                                      "construct PerceptionEncoder(cfg, model=<CLIP with encode_image>)")
        return self.model.encode_image(x, normalize=self.normalize_feature)

    @torch.no_grad()
    def forward(self, videos: List[torch.Tensor]) -> torch.Tensor:
        """vision_encoder.py:47-69 — list of [T_i, 3, H, W] -> [B, max T_i, dim], zero-padded."""
        result = []
        for video in videos:
            video = self.transform(video)
            if self.batch_size > 0 and video.size(0) > self.batch_size:
                res = [self.encode(video[i: i + self.batch_size]) for i in range(0, video.size(0), self.batch_size)]
                result.append(torch.cat(res, dim=0))
            else:
                result.append(self.encode(video))
        return torch.nn.utils.rnn.pad_sequence(result, batch_first=True, padding_value=0.0)
