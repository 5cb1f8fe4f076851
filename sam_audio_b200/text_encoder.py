"""Text conditioning: T5 encoder wrapper (reference: sam_audio/model/text_encoder.py:11-37).

Tokenisation stays on the host (HF tokenizer); on an H100 the encoder stack itself
runs natively through ``sab_t5_forward`` (SURVEY.md §8a a5 / §8f-3 "next" row:
T5LayerNorm, un-scaled attention with the bucketed relative-position bias and
DenseReluDense on the same wgmma GEMM as the DiT), checked against
``transformers.T5EncoderModel`` in tests/test_gpu_parity.py.  The HF module is kept
only as the weight container (``from_pretrained`` / ``state_dict``); its forward is never called here.  When no ``t5-base``
checkpoint/tokenizer is on disk (this sandbox has no network) the same module
graph is built from the t5-base *shape* with seeded random weights and a
deterministic hash tokenizer, so that benchmarks pay the real encoder cost on
synthetic text.
"""
from __future__ import annotations

from typing import List, Tuple

import math

import torch

from .config import T5EncoderConfig


def t5_relative_buckets(L: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """T5's bidirectional relative-position bucket of (key - query) for deltas -(L-1)..L-1, computed with the
    same fp32 torch expression as transformers' T5Attention._relative_position_bucket so that boundary cases
    round identically."""
    rp = torch.arange(-(L - 1), L, dtype=torch.long)
    nb = num_buckets // 2
    buckets = (rp > 0).to(torch.long) * nb
    rp = rp.abs()
    max_exact = nb // 2
    large = max_exact + (torch.log(rp.float() / max_exact) / math.log(max_distance / max_exact)
                         * (nb - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, nb - 1))
    return (buckets + torch.where(rp < max_exact, rp, large)).to(torch.int32)


class _HashTokenizer:
    """Whitespace tokens -> stable ids in [3, vocab); id 1 = </s>, id 0 = pad (T5 conventions)."""

    def __init__(self, vocab_size: int = 32128):
        self.vocab_size = vocab_size

    def __call__(self, texts: List[str], truncation=True, max_length=512, padding="longest", return_tensors="pt"):
        rows = []
        for t in texts:
            ids = []
            for tok in t.split():
                h = 0
                for ch in tok:
                    h = (h * 131 + ord(ch)) % 1000003
                ids.append(3 + h % (self.vocab_size - 3))
            ids = ids[: (max_length or 512) - 1] + [1]
            rows.append(ids)
        width = max(len(r) for r in rows)
        input_ids = torch.zeros(len(rows), width, dtype=torch.long)
        mask = torch.zeros(len(rows), width, dtype=torch.long)
        for i, r in enumerate(rows):
            input_ids[i, : len(r)] = torch.tensor(r)
            mask[i, : len(r)] = 1
        return {"input_ids": input_ids, "attention_mask": mask}


class T5TextEncoder(torch.nn.Module):
    def __init__(self, cfg: T5EncoderConfig, allow_random_init: bool = False, seed: int = 0):
        super().__init__()
        import transformers
        self.pad_mode = cfg.pad_mode
        self.max_length = cfg.max_length
        self.random_init = False
        exc = None
        # the local cache first (no network round trip), then a normal download like the reference does
        # (text_encoder.py:13-14); only if both fail is the checkpoint really unavailable
        for local_only in (True, False):
            try:
                self.model = transformers.T5EncoderModel.from_pretrained(cfg.name, local_files_only=local_only)
                self.tokenizer = transformers.AutoTokenizer.from_pretrained(cfg.name, local_files_only=local_only)
                exc = None
                break
            except Exception as err:  # not cached / no network
                exc = err
        if exc is not None:
            if not allow_random_init:
                raise RuntimeError(
                    f"text encoder '{cfg.name}' is neither cached locally nor downloadable ({type(exc).__name__}); "
                    "pass allow_random_init=True for synthetic benchmarking") from exc
            t5 = transformers.T5Config(vocab_size=32128, d_model=cfg.dim, d_kv=64, d_ff=3072, num_layers=12,
                                       num_heads=12, relative_attention_num_buckets=32, dropout_rate=0.0,
                                       feed_forward_proj="relu")
            with torch.random.fork_rng(devices=[]):
                torch.manual_seed(seed)
                self.model = transformers.T5EncoderModel(t5)
            self.tokenizer = _HashTokenizer(t5.vocab_size)
            self.random_init = True
        self.model.eval()
        self._native = None
        self._native_device = None

    def _engine(self, device):
        from . import _capi
        if self._native is None or self._native_device != device:
            if self._native is not None:
                self._native.close()
            idx = device.index if device.index is not None else torch.cuda.current_device()
            with torch.cuda.device(idx):
                self._native = _capi.T5Engine(self.model.config, idx)
                self._native.load_state_dict(self.model.state_dict())
            self._native_device = device
        return self._native

    @torch.inference_mode()
    def forward(self, texts: List[str]) -> Tuple[torch.Tensor, torch.Tensor]:
        device = next(self.model.parameters()).device
        enc = self.tokenizer(texts, truncation=True, max_length=self.max_length, padding=self.pad_mode,
                             return_tensors="pt")
        input_ids = enc["input_ids"].to(device)
        attention_mask = enc["attention_mask"].to(device)
        if device.type != "cuda":
            raise RuntimeError("T5TextEncoder runs on an H100 only: move the model to cuda first (no CPU path)")
        B, L = input_ids.shape
        eng = self._engine(device)
        cfg = self.model.config
        buckets = t5_relative_buckets(L, cfg.relative_attention_num_buckets,
                                      cfg.relative_attention_max_distance).to(device)
        hidden = torch.empty(B, L, cfg.d_model, device=device, dtype=torch.float32)
        eng.forward(input_ids.long().contiguous(), attention_mask.to(torch.uint8).contiguous(), buckets, hidden)
        return hidden, attention_mask.bool()


class SyntheticTextEncoder(torch.nn.Module):
    """Deterministic stand-in used by parity tests: the same features the oracle sees
    (sam_audio_b200.synthetic.synthetic_text_features), moved to the model's device."""

    def __init__(self, dim: int = 768):
        super().__init__()
        self.dim = dim
        self.register_buffer("_anchor", torch.zeros(1), persistent=False)

    def forward(self, texts: List[str]):
        from .synthetic import synthetic_text_features
        f, m = synthetic_text_features(texts, self.dim)
        return f.to(self._anchor.device), m.to(self._anchor.device)
