"""Streaming separation: ``SAMAudio.stream()`` separates audio pushed in chunks (DESIGN.md section 3).

A stream is solved as windows of W latent frames that start every H = W - W // 8 frames (sam_audio_b200.windows), on
the same library calls as ``separate()``:

- encode: the frames a window adds are encoded from their samples plus the encoder's halo on each side
  (``sab_codec_tiling``); the first slice starts at sample 0 and the last ends at the stream's end, where the codec's
  zero fill is the clip edge as in an un-tiled encode, so the features equal those of the whole recording;
- solve: each window is prepared and solved as a clip of W frames with the stream's text; windows made ready by one
  push are solved as one group;
- blend: the frames that became final are cross-faded from the last two solved windows by ``sab_blend_windows`` into
  an output of just those frames (window starts relative to the first of them);
- decode: final frames are decoded with the decoder's halo of final frames on each side, and only the middle is kept.

The noise of frame t is row t % H of block t // H, drawn from a generator seeded by (seed, block): overlapping windows
start from the same noise rows, and nothing depends on how the input was chunked.  Device memory stays bounded by the
window length, whatever the stream's length: two windows of latents, about W plus two halos of samples and features,
and the engine's cached plans.  PyTorch only allocates, slices and concatenates here; the arithmetic runs in
libsamaudio_b200.so.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import List

import torch

from . import _capi
from .windows import (stream_emit_end, stream_final_frames, stream_frames_available, stream_hop,
                      stream_window_starts, stream_windows_ready, window_groups, window_ramp, window_rows_budget)

_NULL_ANCHOR_IDS = (0, 3)   # the processor's ids of a clip without anchors: <null>, <pad> (processor.py)


@dataclass
class StreamOutput:
    target: torch.Tensor     # [S] samples of the separated source that became final with this call
    residual: torch.Tensor   # [S] the rest of the mixture over the same samples


def _block_seed(seed: int, block: int) -> int:
    """splitmix64 of (seed, block): a distinct generator seed per noise block."""
    z = ((int(seed) & 0xFFFFFFFF) << 32 | (int(block) & 0xFFFFFFFF)) + 0x9E3779B97F4A7C15
    z &= (1 << 64) - 1
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & ((1 << 64) - 1)
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & ((1 << 64) - 1)
    return (z ^ (z >> 31)) & ((1 << 63) - 1)


def stream_noise(seed: int, f0: int, f1: int, block: int, channels: int = 256, device="cuda") -> torch.Tensor:
    """Initial noise of frames [f0, f1) of a stream, [f1 - f0, channels] fp32: frame t is row t % block of block
    t // block, and a block is torch.randn(block, channels) from a generator seeded by (seed, block index).  A pure
    function of (seed, frame), so a window's noise rows and the whole recording's noise agree wherever they overlap."""
    b0, b1 = f0 // block, -(-f1 // block)
    rows = []
    for b in range(b0, b1):
        g = torch.Generator(device=device).manual_seed(_block_seed(seed, b))
        rows.append(torch.randn(block, channels, generator=g, device=device, dtype=torch.float32))
    return torch.cat(rows)[f0 - b0 * block:f1 - b0 * block]


class SeparationStream:
    """Returned by ``SAMAudio.stream()``; see there.  ``push`` returns the samples that became final, ``flush`` the
    rest, and the concatenation of everything returned is ceil(n / hop) * hop samples for n samples pushed."""

    def __init__(self, model, description: str, W: int, seed: int, n_steps: int, method: str):
        self.model = model
        eng = model._ensure_engine()
        cc = model.cfg.audio_codec
        self.W, self.O, self.H = W, window_ramp(W), stream_hop(W)
        self.hop = cc.hop_length
        self.C = 2 * cc.codebook_dim
        self.seed, self.n_steps, self.method = seed, n_steps, method
        self.device = model._device
        self.halo_enc, _ = eng.codec_tiling(False, W)
        self.halo_dec, _ = eng.codec_tiling(True, W)
        # with an encoder halo, no window before flush() reaches the last frame, so flush() always solves the window
        # that carries the stream's end (WIN_LAST)
        assert self.halo_enc >= 1
        with torch.cuda.device(self.device):
            tf, tm = model.text_encoder([description])          # encoded once for the whole stream
        self._text = tf.to(self.device, torch.float32).contiguous()
        self._text_mask = tm.to(self.device).contiguous()
        self._ids = torch.tensor([_NULL_ANCHOR_IDS], dtype=torch.long, device=self.device)
        # samples [wav0, n) live in _buf[:n - wav0]; _spare has the same size and takes the kept samples on a trim
        self._buf = self._spare = None
        self._wav0 = 0
        self.n_samples = 0
        self._enc_end = 0                                      # frames [0, _enc_end) are encoded ...
        self._feat0 = 0                                        # ... and [_feat0, _enc_end) are kept in _feat
        self._feat = torch.empty(0, self.C, device=self.device)
        self.windows_solved = 0
        self._prev = None                                      # latent of window windows_solved - 1, [W, C]
        self.final_frames = 0                                  # frames [0, final_frames) are blended ...
        self._lat0 = 0                                         # ... and [_lat0, final_frames) are kept in _lat
        self._lat = torch.empty(0, self.C, device=self.device)
        self.emitted_frames = 0
        self.closed = False

    # ------------------------------------------------------------------ public
    @torch.inference_mode()
    def push(self, chunk: torch.Tensor) -> StreamOutput:
        """Append samples ([S] or [1, S], S >= 1) and return the samples that became final."""
        self._check_open()
        if chunk.dim() == 2 and chunk.shape[0] == 1:
            chunk = chunk[0]
        if chunk.dim() != 1 or chunk.numel() < 1:
            raise ValueError(f"push() takes [S] or [1, S] samples with S >= 1, got shape {tuple(chunk.shape)}")
        x = chunk.to(device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            self._append(x)
            avail = stream_frames_available(self.n_samples, self.hop, self.halo_enc)
            k1 = stream_windows_ready(avail, self.W)
            return self._advance(k1, flushed=False)

    @torch.inference_mode()
    def flush(self) -> StreamOutput:
        """End the stream: solve the windows that cover the rest (the last padded past the end as in a padded batch),
        return every sample not returned yet, and close the stream."""
        self._check_open()
        self.closed = True
        with torch.cuda.device(self.device):
            if self.n_samples == 0:
                return self._output([])
            T = -(-self.n_samples // self.hop)
            self.n_final = T
            out = self._advance(len(stream_window_starts(T, self.W)), flushed=True)
        self._buf = self._spare = self._feat = self._lat = self._prev = None
        return out

    def workspace_bytes(self) -> int:
        return self.model._ensure_engine().workspace_bytes()

    # ------------------------------------------------------------------ steps
    def _check_open(self):
        if self.closed:
            raise RuntimeError("the stream is closed: flush() has been called")

    def _append(self, x: torch.Tensor):
        held, S = self.n_samples - self._wav0, x.numel()
        if self._buf is None or held + S > self._buf.numel():
            cap = max(held + S, (self.W + 2 * self.halo_enc) * self.hop + S)
            buf = torch.empty(cap, device=self.device, dtype=torch.float32)
            if held:
                buf[:held].copy_(self._buf[:held])
            self._buf, self._spare = buf, torch.empty_like(buf)
        self._buf[held:held + S].copy_(x)
        self.n_samples += S

    def _trim_samples(self):
        """Drop the samples no later encode reads: the next one starts halo_enc frames before _enc_end."""
        keep0 = max(0, self._enc_end - self.halo_enc) * self.hop
        if keep0 <= self._wav0:
            return
        a, b = keep0 - self._wav0, self.n_samples - self._wav0
        self._spare[:b - a].copy_(self._buf[a:b])
        self._buf, self._spare = self._spare, self._buf
        self._wav0 = keep0

    def _encode(self, f1: int, flushed: bool):
        """Encode frames [_enc_end, f1) into _feat.  The encoder reads halo_enc frames of samples on each side; at the
        stream's start the slice starts at sample 0, at flush() it ends at the (reflect-padded) end of the stream."""
        a = self._enc_end
        if f1 <= a:
            return
        s0 = max(0, a - self.halo_enc)
        if flushed:
            wav = self.model._pad(self._buf[s0 * self.hop - self._wav0:self.n_samples - self._wav0].view(1, -1))
            s1 = f1
        else:
            s1 = f1 + self.halo_enc
            wav = self._buf[s0 * self.hop - self._wav0:s1 * self.hop - self._wav0].view(1, -1)
        assert wav.shape[1] == (s1 - s0) * self.hop
        feats = torch.empty(1, s1 - s0, self.C, device=self.device, dtype=torch.float32)
        self.model._ensure_engine().encode(wav.contiguous(), feats)
        self._feat = torch.cat([self._feat, feats[0, a - s0:f1 - s0]])
        self._enc_end = f1

    def _advance(self, k_end: int, flushed: bool) -> StreamOutput:
        """Solve windows [windows_solved, k_end) group by group, blending and decoding what each group makes final."""
        W, H = self.W, self.H
        pieces: List[torch.Tensor] = []
        k0 = self.windows_solved
        groups = window_groups(k_end - k0, 1, W, window_rows_budget())
        for g0, g1 in groups:
            ka, kb = k0 + g0, k0 + g1
            if flushed:
                self._encode(self.n_final, True)
            else:
                for k in range(ka, kb):                        # one fixed-shape encode per window
                    self._encode(k * H + W, False)
            self._solve(ka, kb, flushed and kb == k_end, k_end)
            pieces.append(self._decode(flushed and kb == k_end))
        if not flushed:
            self._trim_samples()
        return self._output(pieces)

    def _solve(self, ka: int, kb: int, last_group: bool, k_end: int):
        """Prepare and solve windows [ka, kb) as one batch of clips of W frames, then blend the frames they make final
        from them and the previously solved window."""
        eng = self.model._ensure_engine()
        W, H, C, dev = self.W, self.H, self.C, self.device
        g = kb - ka
        n_valid = self.n_final if last_group else None
        need = (kb - 1) * H + W                                # features of frames [ka * H, need)
        if need > self._enc_end:                               # past the end of the stream: zero, under the pad mask
            self._feat = torch.cat([self._feat, torch.zeros(need - self._enc_end, C, device=dev)])
            self._enc_end = need
        f = self._feat
        feats = torch.stack([f[k * H - self._feat0:k * H - self._feat0 + W] for k in range(ka, kb)])
        pad = torch.ones(g, W, dtype=torch.bool, device=dev)
        align = torch.zeros(g, W, dtype=torch.long, device=dev)
        if n_valid is not None:
            for i, k in enumerate(range(ka, kb)):
                v = max(0, n_valid - k * H)
                pad[i, v:] = False
                align[i, v:] = 1                               # the processor's <pad> alignment for pad frames
        self.model._install_conditioning(feats, self._text.expand(g, -1, -1), self._text_mask.expand(g, -1), None,
                                         self._ids.expand(g, -1), align, pad, candidates=1)
        n_prev = 0 if self._prev is None else 1
        win = torch.empty(n_prev + g, W, C, device=dev, dtype=torch.float32)
        if n_prev:
            win[0].copy_(self._prev)
        for i, k in enumerate(range(ka, kb)):
            win[n_prev + i].copy_(stream_noise(self.seed, k * H, k * H + W, H, C, dev))
        rows = win[n_prev:]
        eng.solve(rows, self.n_steps, rows, self.method)
        self.windows_solved = kb
        # blend the frames that became final; starts are relative to the first of them
        f_old = self.final_frames
        f_new = stream_final_frames(kb, W, self.n_final if last_group else -1)
        ks = list(range(ka - n_prev, kb))
        seq = torch.zeros(len(ks), dtype=torch.int32, device=dev)
        start = torch.tensor([k * H - f_old for k in ks], dtype=torch.int32, device=dev)
        flags = torch.tensor([_capi.WIN_FIRST * (k == 0) + _capi.WIN_LAST * (last_group and k == k_end - 1) for k in ks],
                             dtype=torch.uint8, device=dev)
        out = torch.empty(1, f_new - f_old, C, device=dev, dtype=torch.float32)
        _capi.blend_windows(win, seq, start, flags, self.O, out)
        self._lat = torch.cat([self._lat, out[0]])
        self.final_frames = f_new
        self._prev = win[-1]
        # the next window reads features from frame kb * H on
        drop = min(kb * H, self._enc_end) - self._feat0
        self._feat = self._feat[drop:].clone()
        self._feat0 += drop

    def _decode(self, flushed: bool) -> torch.Tensor:
        """Decode frames [emitted_frames, emit_end) from the final latent with halo_dec frames on each side; returns
        [2, samples] (target, residual)."""
        a, F = self.emitted_frames, self.final_frames
        b = stream_emit_end(F, self.halo_dec, flushed)
        if b <= a:
            return torch.empty(2, 0, device=self.device)
        d0, d1 = max(0, a - self.halo_dec), F if flushed else b + self.halo_dec
        lat = self._lat[d0 - self._lat0:d1 - self._lat0].unsqueeze(0).contiguous()
        wav = torch.empty(1, 2, (d1 - d0) * self.hop, device=self.device, dtype=torch.float32)
        self.model._ensure_engine().decode(lat, 1, d1 - d0, wav)
        self.emitted_frames = b
        keep0 = max(0, b - self.halo_dec)                        # the next decode reads from here on
        self._lat = self._lat[keep0 - self._lat0:].clone()
        self._lat0 = keep0
        return wav[0, :, (a - d0) * self.hop:(b - d0) * self.hop]

    def _output(self, pieces: List[torch.Tensor]) -> StreamOutput:
        if not pieces:
            e = torch.empty(0, device=self.device, dtype=torch.float32)
            return StreamOutput(target=e, residual=e.clone())
        w = pieces[0] if len(pieces) == 1 else torch.cat(pieces, 1)
        return StreamOutput(target=w[0], residual=w[1])
