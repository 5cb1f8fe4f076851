"""Configuration objects for the H100 SAM-Audio separation path.

Mirrors the JSON schema of the reference's ``config.json``
(reference: sam_audio/model/config.py:10-41 DACVAEConfig, :49-61 T5EncoderConfig,
:86-130 TransformerConfig, :204-231 SAMAudioConfig) so that a checkpoint
directory written for the reference loads here unchanged.  Only the keys the
separate() hot path consumes are interpreted; ranker / judge sections are
carried through verbatim (out of scope, see DESIGN.md).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field, asdict
from typing import Any, Dict, List, Optional


@dataclass
class DACVAEConfig:
    encoder_dim: int = 64
    encoder_rates: List[int] = field(default_factory=lambda: [2, 8, 10, 12])
    latent_dim: int = 1024
    decoder_dim: int = 1536
    decoder_rates: List[int] = field(default_factory=lambda: [12, 10, 8, 2])
    n_codebooks: int = 16
    codebook_size: int = 1024
    codebook_dim: int = 128
    quantizer_dropout: bool = False
    sample_rate: int = 48_000
    mean: float = 0.0
    std: float = 1.0

    @property
    def hop_length(self) -> int:
        return int(math.prod(self.encoder_rates))


@dataclass
class T5EncoderConfig:
    name: str = "t5-base"
    max_length: Optional[int] = 512
    pad_mode: str = "longest"
    dim: int = 768


@dataclass
class PerceptionEncoderConfig:
    dim: int = 1024
    batch_size: int = 300
    name: str = "PE-Core-L14-336"
    normalize_feature: bool = True
    interpolation_mode: str = "BICUBIC"
    image_size: int = 336


@dataclass
class TransformerConfig:
    dim: int = 2048
    n_heads: int = 16
    n_layers: int = 16
    dropout: float = 0.1
    norm_eps: float = 1.0e-05
    qk_norm: bool = True
    fc_bias: bool = False
    ffn_exp: int = 4
    ffn_dim_multiplier: int = 1
    multiple_of: int = 64
    non_linearity: str = "swiglu"
    use_rope: bool = True
    max_positions: int = 10000
    frequency_embedding_dim: int = 256
    timestep_non_linearity: str = "swiglu"
    t_block_non_linearity: str = "silu"
    t_block_bias: bool = True
    context_dim: int = 2048
    context_non_linearity: str = "swiglu"
    context_embedder_dropout: float = 0.0
    context_norm: bool = False
    out_channels: int = 256
    in_channels: Optional[int] = None

    @property
    def head_dim(self) -> int:
        return self.dim // self.n_heads

    @property
    def ffn_hidden(self) -> int:
        """SwiGLU hidden width (reference: transformer.py:179-185)."""
        hidden = int(self.ffn_exp * self.dim)
        if self.non_linearity == "swiglu":
            hidden = int(2 * hidden / 3)
        hidden = int(self.ffn_dim_multiplier * hidden)
        m = self.multiple_of
        return m * ((hidden + m - 1) // m)

    @property
    def rope_theta(self) -> float:
        """reference: transformer.py:405-406."""
        return float(max(10000, 2 * self.max_positions))

    def check_supported(self) -> None:
        """The CUDA path implements the reference's shipped defaults; anything
        else fails loudly instead of silently computing something different."""
        problems = []
        if self.head_dim != 128:
            problems.append(f"head_dim={self.head_dim} (kernels are built for 128)")
        if self.dim % 128:
            problems.append(f"dim={self.dim} not a multiple of 128")
        if self.non_linearity != "swiglu" or self.timestep_non_linearity != "swiglu" \
                or self.context_non_linearity != "swiglu":
            problems.append("non-swiglu projection")
        if self.t_block_non_linearity != "silu":
            problems.append("t_block_non_linearity != silu")
        if not self.qk_norm or not self.use_rope:
            problems.append("qk_norm/use_rope disabled")
        if self.fc_bias or not self.t_block_bias or self.context_norm:
            problems.append("fc_bias/t_block_bias/context_norm variant")
        if self.in_channels is not None:
            problems.append("in_channels data_proj variant")
        if self.context_dim != self.dim:
            problems.append("context_dim != dim")
        if self.frequency_embedding_dim != 256 or self.out_channels != 256:
            problems.append("frequency_embedding_dim/out_channels != 256")
        if problems:
            raise NotImplementedError(
                "sam_audio_b200: unsupported TransformerConfig: " + "; ".join(problems))


class SAMAudioConfig:
    """reference: sam_audio/model/config.py:204-231 (same constructor keys)."""

    def __init__(
        self,
        in_channels: int = 768,
        audio_codec: Optional[Dict[str, Any]] = None,
        text_encoder: Optional[Dict[str, Any]] = None,
        vision_encoder: Optional[Dict[str, Any]] = None,
        transformer: Optional[Dict[str, Any]] = None,
        num_anchors: int = 3,
        anchor_embedding_dim: int = 128,
        visual_ranker: Optional[Dict[str, Any]] = None,
        text_ranker: Optional[Dict[str, Any]] = None,
        span_predictor: Optional[str] = "pe-a-frame-large",
    ):
        self.in_channels = in_channels
        self.audio_codec = DACVAEConfig(**(audio_codec or {}))
        self.text_encoder = T5EncoderConfig(**(text_encoder or {}))
        self.vision_encoder = PerceptionEncoderConfig(**(vision_encoder or {}))
        self.transformer = TransformerConfig(**(transformer or {}))
        self.num_anchors = num_anchors
        self.anchor_embedding_dim = anchor_embedding_dim
        # rankers are post-hoc scoring models outside the hot path (DESIGN.md);
        # the raw dicts are kept so a config round-trips.
        self.visual_ranker = visual_ranker
        self.text_ranker = text_ranker
        self.span_predictor = span_predictor

    def to_dict(self) -> Dict[str, Any]:
        return {
            "in_channels": self.in_channels,
            "audio_codec": asdict(self.audio_codec),
            "text_encoder": asdict(self.text_encoder),
            "vision_encoder": asdict(self.vision_encoder),
            "transformer": asdict(self.transformer),
            "num_anchors": self.num_anchors,
            "anchor_embedding_dim": self.anchor_embedding_dim,
            "visual_ranker": self.visual_ranker,
            "text_ranker": self.text_ranker,
            "span_predictor": self.span_predictor,
        }


# Shape stand-ins for the gated HF configs (SURVEY.md §8d / BASELINE.md §3):
# the per-size config.json files are not in the reference repo.
STAND_IN_TRANSFORMERS: Dict[str, Dict[str, int]] = {
    "sam-audio-small": dict(dim=1536, n_heads=12, n_layers=12, context_dim=1536),
    "sam-audio-base": dict(dim=2048, n_heads=16, n_layers=16, context_dim=2048),
    "sam-audio-large": dict(dim=2816, n_heads=22, n_layers=24, context_dim=2816),
    # tiny shapes for tests / smoke (head_dim stays 128)
    "sam-audio-tiny": dict(dim=256, n_heads=2, n_layers=2, context_dim=256),
}


def stand_in_config(name: str, **overrides) -> SAMAudioConfig:
    if name not in STAND_IN_TRANSFORMERS:
        raise KeyError(f"unknown stand-in model {name!r}; have {sorted(STAND_IN_TRANSFORMERS)}")
    tr = dict(STAND_IN_TRANSFORMERS[name])
    tr.update(overrides.pop("transformer", {}))
    return SAMAudioConfig(transformer=tr, span_predictor=None, **overrides)
