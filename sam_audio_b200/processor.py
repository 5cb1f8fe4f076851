"""Host-side input preparation: SAMAudioProcessor / Batch.

Drop-in mirror of the reference's processor surface (reference:
sam_audio/processor.py:23-36 batch_audio, :39-124 Batch, :127-128 mask_from_sizes,
:158-260 Processor/SAMAudioProcessor).  Pure host code; its integer outputs
(``sizes``, ``audio_pad_mask``, ``anchor_ids``, ``anchor_alignment``) are
bit-exact with the reference (tests/test_processor.py against tests/golden).
"""
from __future__ import annotations

import json
import math
import os
from typing import List, Optional, Sequence, Tuple, Union

import torch

from .config import SAMAudioConfig

Anchor = Tuple[str, float, float]
AudioLike = Union[str, torch.Tensor]

_ANCHOR_IDS = {"<null>": 0, "+": 1, "-": 2, "<pad>": 3}


def _load_audio_file(path: str, sr: int) -> torch.Tensor:
    import torchaudio  # file decoding is outside the hot path (reference processor.py:28-31)
    wav, file_sr = torchaudio.load(path)
    if file_sr != sr:
        wav = torchaudio.functional.resample(wav, file_sr, sr)
    return wav


def batch_audio(audios: Sequence[AudioLike], audio_sampling_rate: int = 48_000):
    """Channel-mean mono mix, right zero-pad to the longest clip -> ([B,1,S], lengths int64).
    The mean is written straight into the padded batch (one pass over the samples); if every input is pinned the
    batch is allocated pinned too, so ``Batch.to("cuda")`` is a single asynchronous copy."""
    wavs = [_load_audio_file(a, audio_sampling_rate) if isinstance(a, str) else a for a in audios]
    lengths = torch.tensor([w.size(-1) for w in wavs])
    longest = int(lengths.max()) if len(wavs) else 0
    pinned = len(wavs) > 0 and all(w.device.type == "cpu" and w.is_pinned() for w in wavs)
    ref = wavs[0]
    out = torch.zeros(len(wavs), 1, longest, dtype=ref.dtype, device=ref.device, pin_memory=pinned)
    for i, w in enumerate(wavs):
        if w.size(0) == 1:
            out[i, 0, : w.size(-1)].copy_(w[0])          # mean over one channel is the channel itself (bit-exact)
        else:
            torch.mean(w, 0, out=out[i, 0, : w.size(-1)])
    return out, lengths


def mask_from_sizes(sizes: torch.Tensor) -> torch.Tensor:
    """True for real frames: frame index < size."""
    steps = torch.arange(sizes.max())
    return steps.unsqueeze(0).expand(len(sizes), -1) < sizes.unsqueeze(1)


class Batch:
    """Mutable container handed to ``SAMAudio.separate`` (same fields as the reference)."""

    def __init__(self, audios, sizes, wav_sizes, descriptions, hop_length, audio_sampling_rate,
                 anchors=None, audio_pad_mask=None, masked_video=None):
        self.audios = audios
        self.sizes = sizes
        self.wav_sizes = wav_sizes
        self.descriptions = descriptions
        self.audio_pad_mask = audio_pad_mask
        self.masked_video = masked_video
        self.hop_length = hop_length
        self.audio_sampling_rate = audio_sampling_rate
        self.process_anchors(anchors)
        assert self.audios.size(0) == len(self.descriptions)

    def _wav_to_feature_idx(self, wav_idx: float) -> int:
        return math.ceil(wav_idx / self.hop_length)       # python double, as the reference

    def to(self, device):
        for name in ("audios", "anchor_ids", "anchor_alignment", "sizes", "wav_sizes"):
            setattr(self, name, getattr(self, name).to(device))
        if self.audio_pad_mask is not None:
            self.audio_pad_mask = self.audio_pad_mask.to(device)
        if self.masked_video is not None:
            self.masked_video = [v.to(device) for v in self.masked_video]
        return self

    def process_anchors(self, anchors: Optional[List[List[Anchor]]]):
        """Token ids per clip ([<null>, <pad>, anchors...]) and, per latent frame, the index into
        that id list: 0 = <null>, 1 = <pad> (pad frames), k>=2 = the k-th anchor covering the frame
        (later anchors overwrite earlier ones)."""
        n = len(self.audios)
        frames = self.audio_pad_mask.size(-1)
        alignment = torch.zeros(n, frames, dtype=torch.long)
        alignment[~self.audio_pad_mask.cpu()] = 1         # host tensor: the batch may already live on the GPU
        if anchors is None:
            ids = torch.tensor([[_ANCHOR_IDS["<null>"], _ANCHOR_IDS["<pad>"]]], dtype=torch.long).repeat(n, 1)
        else:
            per_clip = []
            for i, clip_anchors in enumerate(anchors):
                tokens = [_ANCHOR_IDS["<null>"], _ANCHOR_IDS["<pad>"]]
                for token, t_start, t_end in clip_anchors:
                    first = self._wav_to_feature_idx(t_start * self.audio_sampling_rate)
                    last = self._wav_to_feature_idx(t_end * self.audio_sampling_rate)
                    alignment[i, first:last] = len(tokens)
                    tokens.append(_ANCHOR_IDS[token])
                per_clip.append(tokens)
            width = max(len(t) for t in per_clip)
            ids = torch.full((n, width), _ANCHOR_IDS["<pad>"], dtype=torch.long)
            for i, tokens in enumerate(per_clip):
                ids[i, : len(tokens)] = torch.tensor(tokens, dtype=torch.long)
        dev = self.audios.device
        self.anchor_ids = ids.to(dev)
        self.anchor_alignment = alignment.to(dev)
        self.anchors = anchors


def load_video(sizes, videos, feature_idx_to_wav_idx, audio_sampling_rate):
    """One video frame per latent frame (reference processor.py:131-155).  Tensor inputs only:
    file decoding needs torchcodec, which is outside this path."""
    picked = []
    for size, video in zip(sizes, videos):
        if isinstance(video, str):
            raise NotImplementedError("video file decoding (torchcodec) is outside the H100 hot path; pass tensors")
        assert video.size(1) == 3, f"expected NCHW video, found {video.size(1)} channels"
        idx = torch.linspace(0, video.size(0) - 1, int(size)).round().long()
        picked.append(video[idx])
    return picked


class Processor:
    config_cls = None
    revision = None

    def __init__(self, audio_hop_length: int, audio_sampling_rate: int):
        self.audio_hop_length = audio_hop_length
        self.audio_sampling_rate = audio_sampling_rate

    @classmethod
    def _get_config(cls, model_name_or_path: str):
        if os.path.exists(model_name_or_path):
            path = os.path.join(model_name_or_path, "config.json")
        else:
            from huggingface_hub import hf_hub_download
            path = hf_hub_download(repo_id=model_name_or_path, filename="config.json", revision=cls.revision)
        with open(path) as f:
            return cls.config_cls(**json.load(f))

    @classmethod
    def from_pretrained(cls, model_name_or_path: str):
        cfg = cls._get_config(model_name_or_path)
        return cls(audio_hop_length=cfg.audio_codec.hop_length, audio_sampling_rate=cfg.audio_codec.sample_rate)

    def feature_to_wav_idx(self, feature_idx):
        return feature_idx * self.audio_hop_length

    def wav_to_feature_idx(self, wav_idx):
        if torch.is_tensor(wav_idx):
            return torch.ceil(wav_idx / self.audio_hop_length)   # float32 tensor, as the reference
        return math.ceil(wav_idx / self.audio_hop_length)

    def mask_videos(self, videos, masks):
        out = []
        for v, m in zip(videos, masks):
            if isinstance(v, str) or isinstance(m, str):
                raise NotImplementedError("video file decoding (torchcodec) is outside the H100 hot path; pass tensors")
            out.append(v * m.eq(0))
        return out


class SAMAudioProcessor(Processor):
    config_cls = SAMAudioConfig

    def __call__(self, descriptions: List[str], audios: List[AudioLike],
                 anchors: Optional[List[List[Anchor]]] = None,
                 masked_videos: Optional[List[AudioLike]] = None) -> Batch:
        assert len(descriptions) == len(audios)
        assert anchors is None or len(descriptions) == len(anchors)
        assert masked_videos is None or len(descriptions) == len(masked_videos)
        wavs, wav_sizes = batch_audio(audios, self.audio_sampling_rate)
        sizes = self.wav_to_feature_idx(wav_sizes)
        pad_mask = mask_from_sizes(sizes)
        video = None
        if masked_videos is not None:
            video = load_video(sizes, masked_videos, self.feature_to_wav_idx, self.audio_sampling_rate)
        return Batch(audios=wavs, sizes=sizes, wav_sizes=wav_sizes, descriptions=descriptions,
                     hop_length=self.audio_hop_length, audio_sampling_rate=self.audio_sampling_rate,
                     anchors=anchors, audio_pad_mask=pad_mask, masked_video=video)
