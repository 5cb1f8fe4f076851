"""Streaming separation: ``SAMAudio.stream()`` and ``SAMAudio.stream_group()`` separate audio pushed in chunks
(DESIGN.md section 3).

A stream is solved as windows of W latent frames that start every H = W - W // 8 frames (sam_audio_b200.windows), on
the same library calls as ``separate()``.  Streams live in a ``StreamGroup`` (``SAMAudio.stream()`` is a group of one),
and a tick of the group advances the streams it is given with one batched call per step:

- encode: the frames a window adds are encoded from their samples plus the encoder's halo on each side
  (``sab_codec_tiling``); the first slice starts at sample 0 and the last ends at the stream's end, where the codec's
  zero fill is the clip edge as in an un-tiled encode, so the features equal those of the whole recording.  Slices of
  equal length, from any stream, are the items of one ``sab_encode``;
- solve: every window that becomes ready in the tick is prepared and solved as a clip of W frames with its stream's
  text (padded to the group's token count), all of them in one ``sab_prepare`` + ``sab_solve`` per group of
  ``window_groups``;
- blend: the frames that became final are cross-faded from each stream's last solved windows by ``sab_blend_windows``
  into an output of just those frames (window starts relative to the first of them), one output sequence per stream;
- decode: final frames are decoded with the decoder's halo of final frames on each side, and only the middle is kept;
  slices of equal length are the items of one ``sab_decode``.

Each planned call runs at an item count rounded up to a bucket (``windows.stream_bucket``), the spare slots repeating a
live item, so the engine keeps one resident plan per bucket.  An item's result does not depend on the other items of
its call, so a stream's output is bit-identical whatever the other streams of its group do.

The noise of frame t is row t % H of block t // H, drawn from a generator seeded by (seed, block): overlapping windows
start from the same noise rows, and nothing depends on how the input was chunked.  Device memory stays bounded by the
window length, whatever the stream's length: two windows of latents, about W plus two halos of samples and features,
and the engine's resident plans.

A job (``StreamGroup.submit``) is a stream whose whole input is known: it runs in the filler slots of push ticks, with
its encodes and decodes cut into tiles of the steady slice lengths so that it only joins calls the tick makes anyway.

A stream at another rate, or with several channels, is this stream at the codec's rate with a resampler in front of it
and one behind it (sab_resample, sam_audio_b200.resample).  Ingest turns the pushed samples into the codec-rate samples
whose taps have all arrived (the channel mean is taken as the kernel loads them); output resamples the codec-rate
samples that became final into the stream's rate, emitting a sample once all its taps are final.  At flush() both sides
know their lengths and apply the zero fill at the end.  In a tick every stream's ingest is one sab_resample call before
the encode and every stream's output one call after the decode.  Each resampler holds at most K samples plus one push
(K = its table's taps).  A mono stream at the codec's rate has neither.  PyTorch only allocates, slices and
concatenates here; the arithmetic runs in libsamaudio_b200.so.

A stream with keep_channels also brings every channel to the codec's rate (a per-channel resampler, in the same ingest
launch) and runs a multichannel stage between the decode and the output resampler (_Spread, sab_spread_channels,
sam_audio_b200.channels): the mono target and residual define a Wiener mask applied to each channel, and a sample is
emitted once its last frame's inputs are known.  In a tick every such stream's stage is one sab_spread_channels call.
"""
from __future__ import annotations

import weakref
from collections import defaultdict
from dataclasses import dataclass
from typing import Dict, Iterable, List, Mapping

import torch

from . import _capi
from .channels import keep_from, spread_ready
from .resample import check_rate, first_tap, outputs_ready, resampled_length, taps
from .windows import (TickWindows, stream_bucket, stream_drain_bucket, stream_emit_end, stream_final_frames,
                      stream_flush_rows, stream_frames_available, stream_group_capacity, stream_hop, stream_job_admit,
                      stream_job_min_frames, stream_job_slots, stream_steady_slices, stream_tick_groups, stream_tiles,
                      stream_window_starts, stream_windows_ready, window_ramp, window_rows_budget)

_NULL_ANCHOR_IDS = (0, 3)   # the processor's ids of a clip without anchors: <null>, <pad> (processor.py)


@dataclass
class StreamOutput:
    target: torch.Tensor     # [S] samples of the separated source that became final with this call ([C, S] for a
                             # stream or job with keep_channels)
    residual: torch.Tensor   # [S] the rest of the mixture over the same samples ([C, S] likewise)


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


def check_tick(group, streams: List) -> None:
    """The streams of one tick must be distinct open streams of this group (and so share its window length)."""
    seen = set()
    for s in streams:
        if getattr(s, "group", None) is not group:
            raise ValueError("a tick takes the group's own streams: this stream belongs to another group")
        if s.closed:
            raise RuntimeError("the stream is closed: flush() has been called")
        if s.W != group.W:
            raise ValueError(f"stream window of {s.W} frames in a group of {group.W}-frame windows")
        if id(s) in seen:
            raise ValueError("a stream appears twice in one tick")
        seen.add(id(s))


MAX_CHANNELS = 8


def _samples(chunk: torch.Tensor, channels=None, what: str = "push()") -> torch.Tensor:
    """A pushed chunk as [C, S]: [S], [1, S] or [C, S] with 1 <= C <= 8 and S >= 1, and C equal to the channels of the
    stream's earlier pushes (`channels`, None before the first).  `what` names the call in the messages."""
    if not isinstance(chunk, torch.Tensor):
        raise TypeError(f"{what} takes a tensor of samples, got {type(chunk).__name__}")
    if chunk.dim() == 1:
        chunk = chunk[None]
    if chunk.dim() != 2 or chunk.shape[1] < 1 or not 1 <= chunk.shape[0] <= MAX_CHANNELS:
        raise ValueError(f"{what} takes [S], [1, S] or [C, S] samples with 1 <= C <= {MAX_CHANNELS} and S >= 1, got "
                         f"shape {tuple(chunk.shape)}")
    if channels is not None and chunk.shape[0] != channels:
        raise ValueError(f"the stream has {channels} channel(s) (its first push); got a chunk of {chunk.shape[0]}")
    return chunk


class _Resampler:
    """One rate conversion of a stream: the input samples that later outputs still read ([rows, held], inputs
    [first, received)), and the outputs [0, produced) made so far.  mean=True: the rows are channels of one signal and
    the output is their mean resampled; mean=False: each row is a signal of its own.  Holds at most K samples plus one
    push per row."""

    def __init__(self, orig: int, new: int, rows: int, mean: bool, device):
        self.orig, self.new, self.rows, self.mean = orig, new, rows, mean
        self.K = taps(orig, new)[0]
        self.device = device
        self._buf = self._spare = None
        self.first = self.received = self.produced = 0

    def append(self, x: torch.Tensor):
        held, S = self.received - self.first, x.shape[1]
        if self._buf is None or held + S > self._buf.shape[1]:
            buf = torch.empty(self.rows, 2 * (held + S) + self.K, device=self.device, dtype=torch.float32)
            if held:
                buf[:, :held].copy_(self._buf[:, :held])
            self._buf, self._spare = buf, torch.empty_like(buf)
        self._buf[:, held:held + S].copy_(x)
        self.received += S

    def take(self, flushed: bool):
        """(segments, out): the sab_resample segments of the outputs that became computable (all of them once flushed,
        when the input's length is known) and their output tensor [1 if mean else rows, count]."""
        q0 = self.produced
        q1 = max(q0, outputs_ready(self.received, self.orig, self.new, self.received if flushed else None))
        out = torch.empty(1 if self.mean else self.rows, q1 - q0, device=self.device, dtype=torch.float32)
        segs = []
        if q1 > q0:
            seg = dict(orig_rate=self.orig, new_rate=self.new, in_first=self.first,
                       in_count=self.received - self.first, length=self.received if flushed else -1, out_first=q0,
                       out_count=q1 - q0)
            if self.mean:
                segs.append(dict(seg, channels=self.rows, in_=self._buf.data_ptr(),
                                 in_channel_stride=self._buf.shape[1], out=out.data_ptr()))
            else:
                segs += [dict(seg, in_=self._buf[r].data_ptr(), out=out[r].data_ptr()) for r in range(self.rows)]
        self.produced = q1
        return segs, out

    def trim(self):
        """Drop the inputs no later output reads (after the launch that read them is enqueued)."""
        keep0 = min(self.received, max(0, first_tap(self.produced, self.orig, self.new)))
        if keep0 <= self.first:
            return
        a, b = keep0 - self.first, self.received - self.first
        self._spare[:, :b - a].copy_(self._buf[:, a:b])
        self._buf, self._spare = self._spare, self._buf
        self.first = keep0


class _Rows:
    """Samples [first, received) of `rows` signals on the device, in buf[:, :received - first]; spare has the same size
    and takes the kept samples on a trim, so a stream in steady state allocates nothing."""

    def __init__(self, rows: int, device):
        self.rows, self.device = rows, device
        self.buf = self._spare = None
        self.first = self.received = 0

    def append(self, x: torch.Tensor):
        held, S = self.received - self.first, x.shape[1]
        if self.buf is None or held + S > self.buf.shape[1]:
            buf = torch.empty(self.rows, 2 * (held + S), device=self.device, dtype=torch.float32)
            if held:
                buf[:, :held].copy_(self.buf[:, :held])
            self.buf, self._spare = buf, torch.empty_like(buf)
        self.buf[:, held:held + S].copy_(x)
        self.received += S

    def trim(self, keep0: int):
        keep0 = min(self.received, keep0)
        if keep0 <= self.first:
            return
        a, b = keep0 - self.first, self.received - self.first
        self._spare[:, :b - a].copy_(self.buf[:, a:b])
        self.buf, self._spare = self._spare, self.buf
        self.first = keep0

    def ptr(self, row: int = 0) -> int:
        return 0 if self.buf is None else self.buf[row].data_ptr()


class _Spread:
    """The multichannel stage of a keep-channels stream (sab_spread_channels, sam_audio_b200.channels): the codec-rate
    mono target and residual as they become final (tr, 2 rows), the codec-rate channels as they arrive (x, C rows), and
    the outputs [0, produced) made so far.  The lengths are known at flush().  Holds, per row, the samples the next
    output's frames read: the mono stream's delay plus N samples."""

    def __init__(self, C: int, device):
        self.C, self.device = C, device
        self.tr, self.x = _Rows(2, device), _Rows(C, device)
        self.tr_length = self.x_length = None
        self.produced = 0

    def take(self):
        """(segment, out): the sab_spread_channels segment of the outputs that became computable (None if there are
        none) and their output tensor [2, C, count] (target, residual)."""
        q0 = self.produced
        q1 = max(q0, spread_ready(self.tr.received, self.x.received, self.tr_length, self.x_length))
        out = torch.empty(2, self.C, q1 - q0, device=self.device, dtype=torch.float32)
        seg = None
        if q1 > q0:
            tr, x = self.tr, self.x
            seg = dict(channels=self.C, target=tr.ptr(0), residual=tr.ptr(1), tr_first=tr.first,
                       tr_count=tr.received - tr.first, tr_length=-1 if self.tr_length is None else self.tr_length,
                       mix=x.ptr(), mix_channel_stride=0 if x.buf is None else x.buf.shape[1], mix_first=x.first,
                       mix_count=x.received - x.first, mix_length=-1 if self.x_length is None else self.x_length,
                       out_target=out[0].data_ptr(), out_residual=out[1].data_ptr(), out_channel_stride=q1 - q0,
                       out_first=q0, out_count=q1 - q0)
        self.produced = q1
        return seg, out

    def trim(self):
        """Drop the inputs no later output reads (after the launch that read them is enqueued)."""
        k = keep_from(self.produced)
        self.tr.trim(k)
        self.x.trim(k)


class SeparationStream:
    """Returned by ``SAMAudio.stream()`` and ``StreamGroup.open()``; see there.  ``push`` returns the samples that became
    final, ``flush`` the rest, and the concatenation of everything returned is ceil(n / hop) * hop samples for n samples
    pushed.  ``push`` and ``flush`` are ticks of the stream's group with this stream alone."""

    def __init__(self, group: "StreamGroup", description: str, seed: int, sample_rate: int,
                 keep_channels: bool = False):
        self.group = group
        self.model = group.model
        self.sample_rate = sample_rate                         # of push() and of the outputs
        self.keep_channels = keep_channels                     # outputs [C, S]: the stems of every pushed channel
        self.channels = None                                   # of push(), fixed by the first
        self._ingest = None                                    # resampler to the codec's rate (set by the first push)
        self._split = None                                     # keep_channels: per-channel resampler to the codec's rate
        self._spread = None                                    # keep_channels: the multichannel stage (_Spread)
        sr = self.model.sample_rate
        # the output resampler: mono target and residual, or (keep_channels) 2 C rows made at the first push
        self._emit = None if sample_rate == sr or keep_channels else _Resampler(sr, sample_rate, 2, False, group.device)
        self.W, self.O, self.H, self.hop, self.C = group.W, group.O, group.H, group.hop, group.C
        self.seed = seed
        self.device = group.device
        with torch.cuda.device(self.device):
            tf, tm = self.model.text_encoder([description])     # encoded once for the whole stream
        self._text = tf.to(self.device, torch.float32).contiguous()
        self._text_mask = tm.to(self.device).contiguous()
        self.n_tokens = self._text.shape[1]
        # samples [wav0, n) live in _buf[:n - wav0]; _spare has the same size and takes the kept samples on a trim
        self._buf = self._spare = None
        self._wav0 = 0
        self.n_samples = 0
        self.n_final = None                                    # frames of the stream, known at flush()
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
    def push(self, chunk: torch.Tensor) -> StreamOutput:
        """Append samples ([S], [1, S] or [C, S] with 1 <= C <= 8, S >= 1, at the stream's rate) and return the samples
        that became final, at the stream's rate."""
        return self.group.push({self: chunk})[self]

    def flush(self) -> StreamOutput:
        """End the stream: solve the windows that cover the rest (the last padded past the end as in a padded batch),
        return every sample not returned yet, and close the stream."""
        return self.group.flush([self])[self]

    def workspace_bytes(self) -> int:
        return self.model._ensure_engine().workspace_bytes()

    # ------------------------------------------------------------------ state
    def _append(self, x: torch.Tensor):
        held, S = self.n_samples - self._wav0, x.numel()
        if self._buf is None or held + S > self._buf.numel():
            cap = max(held + S, (self.W + 2 * self.group.halo_enc) * self.hop + S)
            buf = torch.empty(cap, device=self.device, dtype=torch.float32)
            if held:
                buf[:held].copy_(self._buf[:held])
            self._buf, self._spare = buf, torch.empty_like(buf)
        self._buf[held:held + S].copy_(x)
        self.n_samples += S

    def _trim_samples(self):
        """Drop the samples no later encode reads: the next one starts halo_enc frames before _enc_end."""
        keep0 = max(0, self._enc_end - self.group.halo_enc) * self.hop
        if keep0 <= self._wav0:
            return
        a, b = keep0 - self._wav0, self.n_samples - self._wav0
        self._spare[:b - a].copy_(self._buf[a:b])
        self._buf, self._spare = self._spare, self._buf
        self._wav0 = keep0

    def _text_at(self, L: int):
        """Text features and mask padded to L tokens (zero features, masked)."""
        n = self.n_tokens
        if n == L:
            return self._text[0], self._text_mask[0]
        f = torch.zeros(L, self._text.shape[2], device=self.device, dtype=torch.float32)
        m = torch.zeros(L, dtype=self._text_mask.dtype, device=self.device)
        f[:n], m[:n] = self._text[0], self._text_mask[0]
        return f, m

    def _ends_at(self, kb: int) -> bool:
        """Window kb - 1 is the stream's last, which carries its end (WIN_LAST, the pad mask past n_final): known once
        the stream's length is, at flush() (a job: from the start)."""
        return self.n_final is not None and kb == len(stream_window_starts(self.n_final, self.W))

    def _release(self):
        self._buf = self._spare = self._feat = self._lat = self._prev = None
        self._ingest = self._emit = self._split = self._spread = None

    def _set_channels(self, C: int):
        if self.channels is None:
            self.channels = C
            sr = self.model.sample_rate
            if self.sample_rate != sr or C > 1:
                self._ingest = _Resampler(self.sample_rate, sr, C, True, self.device)
            if self.keep_channels:
                self._spread = _Spread(C, self.device)
                if self.sample_rate != sr:
                    self._split = _Resampler(self.sample_rate, sr, C, False, self.device)
                    self._emit = _Resampler(sr, self.sample_rate, 2 * C, False, self.device)

    def _output(self, pieces: List[torch.Tensor]) -> StreamOutput:
        if not pieces:
            e = torch.empty(0, device=self.device, dtype=torch.float32)
            return StreamOutput(target=e, residual=e.clone())
        w = pieces[0] if len(pieces) == 1 else torch.cat(pieces, 1)
        return StreamOutput(target=w[0], residual=w[1])


class SeparationJob:
    """Returned by ``StreamGroup.submit()``: a whole recording separated in the idle slots of the group's ticks.  It is
    the stream ``model.stream(description, window_seconds, seed, sample_rate)`` would be with the recording pushed once
    and flushed: the same windows, noise, blend and resamplers, so ``result()`` equals that stream's concatenated output
    bit for bit.  Its encodes and decodes are cut into tiles of the steady slice lengths (windows.stream_tiles).

    It holds the recording at the codec's rate (until it is encoded), the output at the codec's rate as it is decoded
    (at its own rate once done), and a stream's per-window state; features and latents are kept from the next window's
    and the next decode tile's first frame on.  All of it is bounded by its own length."""

    _text_at = SeparationStream._text_at
    _ends_at = SeparationStream._ends_at

    def __init__(self, group: "StreamGroup", description: str, seed: int, sample_rate: int, wav: torch.Tensor,
                 keep_channels: bool = False):
        self._group = weakref.ref(group)      # the group's finalizer cancels its jobs, so a job must not keep it alive
        self.model = group.model
        self.sample_rate = sample_rate
        self.keep_channels = keep_channels
        self.W, self.O, self.H, self.hop, self.C = group.W, group.O, group.H, group.hop, group.C
        self.seed = seed
        self.device = group.device
        with torch.cuda.device(self.device):
            tf, tm = self.model.text_encoder([description])
        self._text = tf.to(self.device, torch.float32).contiguous()
        self._text_mask = tm.to(self.device).contiguous()
        self.n_tokens = self._text.shape[1]
        sr = self.model.sample_rate
        self._x48 = None                                       # keep_channels: the channels at the codec's rate [C, n]
        with torch.cuda.device(self.device):
            if sample_rate != sr or wav.shape[0] > 1:        # the stream's ingest, with the whole length known
                x = wav.to(device=self.device, dtype=torch.float32).contiguous()
                S = x.shape[1]
                x48 = torch.empty(1, resampled_length(S, sample_rate, sr), device=self.device, dtype=torch.float32)
                seg = dict(orig_rate=sample_rate, new_rate=sr, in_first=0, in_count=S, length=S, out_first=0,
                           out_count=x48.shape[1])
                segs = [dict(seg, channels=x.shape[0], in_=x.data_ptr(), in_channel_stride=S, out=x48.data_ptr())]
                if keep_channels and sample_rate != sr:        # ... and the per-channel one, in the same launch
                    self._x48 = torch.empty(x.shape[0], x48.shape[1], device=self.device, dtype=torch.float32)
                    segs += [dict(seg, in_=x[c].data_ptr(), out=self._x48[c].data_ptr()) for c in range(x.shape[0])]
                elif keep_channels:
                    self._x48 = wav.to(device=self.device, dtype=torch.float32, copy=True).contiguous()
                self.model._ensure_engine().resample(segs)
            else:
                # a copy, as push() makes one: the tiles read the recording over later ticks, and the caller may reuse
                # its tensor as soon as submit() returns
                x48 = wav.to(device=self.device, dtype=torch.float32, copy=True).contiguous()
                if keep_channels:
                    self._x48 = x48
            self._wav = self.model._pad(x48)[0]               # reflect-padded to n_final frames, as flush() pads
        self.n_samples = x48.shape[1]
        self._init_schedule(-(-self.n_samples // self.hop), group.halo_enc, group.halo_dec)
        self._feat = torch.empty(0, self.C, device=self.device)
        self._prev = None
        self._lat = torch.empty(0, self.C, device=self.device)
        self._out = torch.empty(2, self.n_final * self.hop, device=self.device, dtype=torch.float32)
        self._result = None
        self.done = self.cancelled = False

    def _init_schedule(self, n_final: int, halo_enc: int, halo_dec: int):
        """The job's tile plans and progress counters for a recording of n_final frames (host state only)."""
        self.n_final = n_final
        self._enc_len, self._dec_len = le, ld = stream_steady_slices(self.W, halo_enc, halo_dec)
        self._enc_tiles = stream_tiles(n_final, le, halo_enc)
        self._dec_tiles = stream_tiles(n_final, ld, halo_dec)
        self._enc_next = self._dec_next = 0                   # tiles done
        self.windows_total = len(stream_window_starts(n_final, self.W))
        self.windows_solved = 0
        self._enc_end = self._feat0 = 0                       # features [0, _enc_end) encoded, [_feat0, ...) kept
        self.final_frames = self._lat0 = 0                    # latents [0, final_frames) final, [_lat0, ...) kept

    # ------------------------------------------------------------------ public
    def result(self) -> StreamOutput:
        """The separated recording at the job's rate: the concatenated target and residual of the stream above."""
        if self.cancelled:
            raise RuntimeError("the job was cancelled")
        if not self.done:
            raise RuntimeError(f"the job is not done ({self.windows_solved} of {self.windows_total} windows solved): "
                               "its group runs it in idle slots of push ticks; group.drain() finishes it")
        return self._result

    def cancel(self) -> None:
        """Stop the job and free its device memory (its result too, if it is done)."""
        self.cancelled = True
        self._release()
        self._result = None
        g = self._group()
        if g is not None and self in g._jobs:
            g._jobs.remove(self)

    # ------------------------------------------------------------------ what the next calls can take
    def _encode_offer(self) -> int:
        return len(self._enc_tiles) - self._enc_next

    def _solve_offer(self) -> int:
        """Windows ready to solve: their features are encoded (the last one's once the whole recording is)."""
        if self._enc_next == len(self._enc_tiles):
            return self.windows_total - self.windows_solved
        return max(0, min(self.windows_total, stream_windows_ready(self._enc_end, self.W)) - self.windows_solved)

    def _decode_offer(self) -> int:
        """Decode tiles whose latent frames are all final."""
        n = 0
        for start, _, _ in self._dec_tiles[self._dec_next:]:
            if start + self._dec_len > self.final_frames:
                break
            n += 1
        return n

    def _release(self):
        self._wav = self._feat = self._lat = self._prev = self._out = self._text = self._text_mask = None
        self._x48 = None


class StreamGroup:
    """Returned by ``SAMAudio.stream_group()``; see there.  Streams of one group share the window length and the ODE
    grid; a tick (``push`` / ``flush``) advances any subset of the open streams with batched library calls."""

    def __init__(self, model, W: int, n_steps: int, method: str, resident_plans: bool):
        self.model = model
        eng = model._ensure_engine()
        cc = model.cfg.audio_codec
        self.W, self.O, self.H = W, window_ramp(W), stream_hop(W)
        self.hop = cc.hop_length
        self.C = 2 * cc.codebook_dim
        self.n_steps, self.method = n_steps, method
        self.device = model._device
        self.halo_enc, _ = eng.codec_tiling(False, W)
        self.halo_dec, _ = eng.codec_tiling(True, W)
        # with an encoder halo, no window before flush() reaches the last frame, so flush() always solves the window
        # that carries the stream's end (WIN_LAST)
        assert self.halo_enc >= 1
        self.capacity = stream_group_capacity(W, window_rows_budget())
        self._steady = stream_steady_slices(W, self.halo_enc, self.halo_dec)   # frames of steady encode/decode slices
        self.L = 0                      # text tokens of every window: the longest prompt opened in the group so far
        self.streams: List[SeparationStream] = []
        self._ids = torch.tensor([_NULL_ANCHOR_IDS], dtype=torch.long, device=self.device)
        self.closed = False
        self._holds_limits = resident_plans
        self._buckets_used = set()     # item counts of the planned calls of push ticks (the residency follows them)
        self._solve_buckets = set()    # ... of their solves: the DiT plans a flush tick reuses
        self._jobs: List[SeparationJob] = []   # submitted and not done, first in first out
        if resident_plans:
            # a group dropped without close() cancels its jobs and gives the residency back when it is collected
            self._limits_key = object()
            self._finalizer = weakref.finalize(self, _drop_group, model._hold_plan_limits, self._limits_key, self._jobs)
            self._finalizer.atexit = False

    # ------------------------------------------------------------------ public
    def open(self, description: str, seed: int = 0, sample_rate=None, keep_channels: bool = False) -> SeparationStream:
        """A new stream of the group with its own prompt and noise seed.  sample_rate: of its pushes and outputs (an
        integer in [8000, 192000] Hz; None: the model's rate).  keep_channels: the outputs are [C, S], the stems of
        every pushed channel (SAMAudio.stream)."""
        if self.closed:
            raise RuntimeError("the stream group is closed")
        if not isinstance(description, str):
            raise TypeError("a stream separates one source: description must be one string")
        keep_channels = check_keep_channels(keep_channels)
        sr = self.model.sample_rate if sample_rate is None else check_rate(sample_rate)
        s = SeparationStream(self, description, int(seed), sr, keep_channels)
        self.L = max(self.L, s.n_tokens)
        self.streams.append(s)
        return s

    @torch.inference_mode()
    def submit(self, wav: torch.Tensor, description: str, seed: int = 0, sample_rate=None,
               keep_channels: bool = False) -> SeparationJob:
        """Queue a whole recording ([S], [1, S] or [C, S] with C <= 8, at sample_rate) to be separated in the idle slots
        of the group's ticks; see SeparationJob.  sample_rate, keep_channels and the prompt are as for open() (the
        prompt counts toward the group's text length: a prompt longer than every earlier one makes the next tick
        re-plan its buckets at the new length, as open() does).  The recording is copied, so the caller may reuse its
        tensor at once.  It must be long enough to be cut into codec tiles of the steady slice lengths
        (stream_job_min_frames)."""
        if self.closed:
            raise RuntimeError("the stream group is closed")
        if not isinstance(description, str):
            raise TypeError("a job separates one source: description must be one string")
        keep_channels = check_keep_channels(keep_channels)
        sr = self.model.sample_rate if sample_rate is None else check_rate(sample_rate)
        x = _samples(wav, what="submit()")
        n48 = x.shape[1] if sr == self.model.sample_rate else resampled_length(x.shape[1], sr, self.model.sample_rate)
        need = stream_job_min_frames(self.W, self.halo_enc, self.halo_dec)
        if -(-n48 // self.hop) < need:
            raise ValueError(f"a job of {x.shape[1] / sr:.3f} s is too short: a stream group's jobs need at least "
                             f"{need * self.hop / self.model.sample_rate:.3f} s ({need} latent frames) at this window "
                             "length; separate() or stream() take shorter recordings")
        job = SeparationJob(self, description, int(seed), sr, x, keep_channels)
        self.L = max(self.L, job.n_tokens)
        self._jobs.append(job)
        return job

    @torch.inference_mode()
    def drain(self, jobs=None) -> None:
        """Run ticks that hold only jobs until the given jobs (default: all) are done.  Jobs are served first in, first
        out, so the jobs submitted before them finish too.  Each planned call runs at a solve bucket the group has
        already used (bucket 1 if it has never ticked), and these ticks are the only ones in which a job may build a
        plan."""
        want = list(self._jobs) if jobs is None else list(jobs)
        for j in want:
            if not isinstance(j, SeparationJob) or j._group() is not self:
                raise ValueError("drain() takes jobs submitted to this group")
        with torch.cuda.device(self.device):
            while any(not (j.done or j.cancelled) for j in want):
                self._tick([], flushed=False, drain=True)

    @torch.inference_mode()
    def push(self, chunks: Mapping[SeparationStream, torch.Tensor]) -> Dict[SeparationStream, StreamOutput]:
        """One tick: append each stream's samples ([S], [1, S] or [C, S], S >= 1, at its rate) and return, per stream,
        the samples that became final, at its rate."""
        streams = list(chunks)
        check_tick(self, streams)
        xs = [_samples(chunks[s], s.channels).to(device=self.device, dtype=torch.float32) for s in streams]
        with torch.cuda.device(self.device):
            for s, x in zip(streams, xs):
                s._set_channels(x.shape[0])
            ingested, split = self._resample_in(streams, xs, flushed=False)
            due = []
            for s, x in zip(streams, xs):
                s._append(ingested.get(s, x[0]))
                if s._spread is not None:
                    s._spread.x.append(split.get(s, x))
                avail = stream_frames_available(s.n_samples, self.hop, self.halo_enc)
                due.append((s, s.windows_solved, stream_windows_ready(avail, self.W)))
            out = self._tick(due, flushed=False)
            for s in streams:
                s._trim_samples()
            out = self._spread_out(out, flushed=False)
            out = self._resample_out(out, flushed=False)
        return out

    @torch.inference_mode()
    def flush(self, streams: Iterable[SeparationStream]) -> Dict[SeparationStream, StreamOutput]:
        """One tick that ends the given streams: each returns every sample not returned yet and is closed."""
        streams = list(streams)
        check_tick(self, streams)
        try:
            with torch.cuda.device(self.device):
                # the ingest's zero fill at the end: the codec-rate stream gets the rest of its samples first
                ingested, split = self._resample_in(streams, [None] * len(streams), flushed=True)
                for s, x in ingested.items():
                    if x.numel():
                        s._append(x)
                for s, x in split.items():
                    if x.numel():
                        s._spread.x.append(x)
                live = [s for s in streams if s.n_samples > 0]
                for s in live:
                    s.n_final = -(-s.n_samples // self.hop)
                out = self._tick([(s, s.windows_solved, len(stream_window_starts(s.n_final, self.W))) for s in live],
                                 flushed=True)
                for s in streams:
                    out.setdefault(s, s._output([]))
                out = self._spread_out(out, flushed=True)
                out = self._resample_out(out, flushed=True)
        finally:
            # a stream is ended whether or not its last tick succeeded: a failed flush leaves no half-advanced stream
            # in the group, so close() still works and gives the engine back its residency
            for s in streams:
                s.closed = True
                s._release()
                self.streams.remove(s)
        return out

    def close(self) -> Dict[SeparationStream, StreamOutput]:
        """Flush every open stream, finish the jobs left (drain()), close the group and give the engine back its
        default plan residency.  Jobs still queued when a tick fails are cancelled."""
        self.closed = True
        try:
            out = self.flush(list(self.streams)) if self.streams else {}
            self.drain()
            return out
        finally:
            for j in list(self._jobs):
                j.cancel()
            self._release_limits()

    def _release_limits(self):
        if self._holds_limits:
            self._holds_limits = False
            self._finalizer.detach()
            self.model._hold_plan_limits(self._limits_key, None)

    def _slots(self, n: int, flushed: bool, solve: bool) -> List[int]:
        """stream_bucket of n items.  A push tick may use a new bucket, and the engine's plan residency is raised to
        the buckets this group has used: one DiT plan per bucket, and per direction two codec slice lengths per bucket
        (a stream's first window and the later ones) plus one for the varying lengths of flushes, which therefore
        replace each other.  A flush tick's solve reuses a bucket already used when one is large enough; its encode and
        decode slices have lengths of their own, so no resident plan fits them and they use no bucket slot."""
        if not self._holds_limits or (flushed and not solve):
            return stream_bucket(n, self.capacity)
        slots = stream_bucket(n, self.capacity, self._solve_buckets if flushed else ())
        self._solve_buckets.add(len(slots))
        if len(slots) not in self._buckets_used:
            self._buckets_used.add(len(slots))
            k = len(self._buckets_used)
            self.model._hold_plan_limits(self._limits_key, (k, 2 * k + 1))
        return slots

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    # ------------------------------------------------------------------ rate conversion
    def _resample_in(self, streams, xs, flushed: bool):
        """Ingest of a tick, one sab_resample call for every stream that has a resampler in front: the codec-rate
        samples that became computable (all the rest at flush()), per stream, as (mono [S] per stream, channels [C, S]
        per keep-channels stream at another rate).  xs: the pushed [C, S] (None at flush)."""
        segs, outs, split = [], {}, {}
        for s, x in zip(streams, xs):
            for r, into in ((s._ingest, outs), (s._split, split)):
                if r is None:
                    continue
                if x is not None:
                    r.append(x)
                sg, out = r.take(flushed)
                segs += sg
                into[s] = out[0] if r.mean else out
        self.model._ensure_engine().resample(segs)
        for s in outs:
            s._ingest.trim()
        for s in split:
            s._split.trim()
        return outs, split

    def _spread_out(self, out: Dict[SeparationStream, StreamOutput], flushed: bool) -> Dict[SeparationStream,
                                                                                           StreamOutput]:
        """The multichannel stage of a tick, one sab_spread_channels call for every keep-channels stream: the codec-rate
        mono samples that became final are appended to its _Spread, and the [C, S] stems whose frames are all
        computable (all the rest at flush(), when both lengths are known) replace them."""
        segs, ys = [], {}
        for s, o in out.items():
            sp = s._spread
            if sp is None:
                continue
            if o.target.numel():
                sp.tr.append(torch.stack([o.target, o.residual]))
            if flushed:
                sp.tr_length, sp.x_length = sp.tr.received, sp.x.received
            seg, ys[s] = sp.take()
            if seg is not None:
                segs.append(seg)
        self.model._ensure_engine().spread_channels(segs)
        for s, y in ys.items():
            s._spread.trim()
            out[s] = StreamOutput(target=y[0], residual=y[1])
        return out

    def _resample_out(self, out: Dict[SeparationStream, StreamOutput], flushed: bool) -> Dict[SeparationStream,
                                                                                             StreamOutput]:
        """Output of a tick, one sab_resample call for every stream that has a resampler behind: the codec-rate samples
        that became final are appended to it, and the stream-rate samples whose taps are all final are returned."""
        segs, ys = [], {}
        for s, o in out.items():
            r = s._emit
            if r is None:
                continue
            if o.target.numel():
                r.append(torch.cat([o.target, o.residual]) if s.keep_channels else torch.stack([o.target, o.residual]))
            sg, ys[s] = r.take(flushed)
            segs += sg
        self.model._ensure_engine().resample(segs)
        for s, y in ys.items():
            s._emit.trim()
            h = y.shape[0] // 2                            # 1, or C with keep_channels
            out[s] = StreamOutput(target=y[:h] if s.keep_channels else y[0], residual=y[h:] if s.keep_channels else y[1])
        return out

    # ------------------------------------------------------------------ the tick
    def _tick(self, due, flushed: bool, drain: bool = False) -> Dict[SeparationStream, StreamOutput]:
        """Solve windows [k0, k_end) of every (stream, k0, k_end) in due, group by group: encode, solve, blend and decode
        what each group makes final.  In a push tick the queued jobs take the filler slots of its calls; a drain tick
        (due empty) holds only jobs, and a flush tick none."""
        pieces: Dict[SeparationStream, List[torch.Tensor]] = {s: [] for s, _, _ in due}
        budget = window_rows_budget()
        if flushed and self._holds_limits:
            budget = stream_flush_rows(budget, self.W, self._solve_buckets)
        jobs = [] if flushed else list(self._jobs)
        for grp in ([[]] if drain else stream_tick_groups(due, self.W, budget)):
            self._encode(grp, flushed, jobs, drain)
            rows, job_windows = self._solve(grp, flushed, jobs, drain)
            if rows is not None:
                self._blend(grp + job_windows, rows)
            for s, piece in self._decode(grp, flushed, jobs, drain):
                pieces[s].append(piece)
        if jobs:
            self._finish_jobs(jobs)
        return {s: s._output(p) for s, p in pieces.items()}

    def _call_slots(self, n_live: int, flushed: bool, solve: bool, jobs, offer, drain: bool):
        """(slots, taken) of one planned call with n_live live items: a push tick's call runs at its bucket (_slots) and
        the jobs take its filler slots, first in first out (stream_job_admit, offer(job) = the job's items ready for
        it); a drain tick's call runs at a resident solve bucket (stream_drain_bucket), or not at all (slots None)
        when no job has an item ready.  taken: the job items of the call, per job."""
        offers = [offer(j) for j in jobs]
        if drain:
            if not any(offers):
                return None, offers
            size = stream_drain_bucket(sum(offers), self._solve_buckets)
        else:
            slots = self._slots(n_live, flushed, solve)
            if not any(offers):
                return slots, [0] * len(jobs)
            size = len(slots)
        taken = stream_job_admit(offers, size - n_live)
        return stream_job_slots(n_live, size, sum(taken)), taken

    def _encode(self, grp, flushed: bool, jobs=(), drain: bool = False):
        """Encode the frames the group's windows need: [_enc_end, k * H + W) per window, or up to the stream's end at
        flush().  A slice reads halo_enc frames of samples on each side; at a stream's start it starts at sample 0, at
        flush() it ends at the (reflect-padded) end of the stream.  Jobs' tiles fill the call of steady slices."""
        hop, halo = self.hop, self.halo_enc
        items = []                                             # (stream, samples, first kept row, end row, new end)
        for w in grp:
            s = w.key
            a = s._enc_end
            for f1 in ([s.n_final] if flushed else [k * self.H + self.W for k in range(w.ka, w.kb)]):
                if f1 <= a:
                    continue
                s0 = max(0, a - halo)
                if flushed:
                    wav = self.model._pad(s._buf[s0 * hop - s._wav0:s.n_samples - s._wav0].view(1, -1))[0]
                    s1 = f1
                else:
                    s1 = f1 + halo
                    wav = s._buf[s0 * hop - s._wav0:s1 * hop - s._wav0]
                assert wav.numel() == (s1 - s0) * hop
                items.append((s, wav, a - s0, f1 - s0, f1))
                a = f1
        by_len = defaultdict(list)
        for i, j in enumerate(items):
            by_len[j[1].numel()].append(i)
        steady = self._steady[0]
        if drain:
            by_len.setdefault(steady * hop, [])                # a drain tick has no live items: make the steady call
        feats = {}
        eng = self.model._ensure_engine()
        for n, idx in by_len.items():
            if n == steady * hop and (jobs or drain):
                slots, taken = self._call_slots(len(idx), flushed, False, jobs, SeparationJob._encode_offer, drain)
                if slots is None:
                    continue
                for j, t in zip(jobs, taken):
                    for start, k0, k1 in j._enc_tiles[j._enc_next:j._enc_next + t]:
                        idx.append(len(items))
                        items.append((j, j._wav[start * hop:(start + steady) * hop], k0 - start, k1 - start, k1))
                    j._enc_next += t
            else:
                slots = self._slots(len(idx), flushed, solve=False)
            wav = torch.stack([items[idx[i]][1] for i in slots])
            out = torch.empty(len(slots), n // hop, self.C, device=self.device, dtype=torch.float32)
            eng.encode(wav, out)
            for i, ji in enumerate(idx):
                feats[ji] = out[i]
        for i, (s, _, r0, r1, f1) in enumerate(items):          # in item order: a stream's slices follow each other
            s._feat = torch.cat([s._feat, feats[i][r0:r1]])
            s._enc_end = f1
        for j in jobs:
            if j._enc_next == len(j._enc_tiles):
                j._wav = None                                  # encoded: the recording is no longer read

    def _solve(self, grp, flushed: bool, jobs=(), drain: bool = False):
        """Prepare and solve the group's windows, then the job windows the call takes, as one batch of clips of W frames.
        Returns their latents [n, W, C] (None when a drain tick has nothing to solve) and the job windows."""
        W, H, C, dev = self.W, self.H, self.C, self.device
        n_live = sum(w.kb - w.ka for w in grp)
        slots, taken = self._call_slots(n_live, flushed, True, jobs, SeparationJob._solve_offer, drain)
        if slots is None:
            return None, []
        job_windows = [TickWindows(j, j.windows_solved, j.windows_solved + t, j._ends_at(j.windows_solved + t))
                       for j, t in zip(jobs, taken) if t]
        feats, texts, masks, pads, aligns, noise = [], [], [], [], [], []
        for w in grp + job_windows:
            s = w.key
            n_valid = s.n_final if s._ends_at(w.kb) else None
            need = (w.kb - 1) * H + W                          # features of frames [ka * H, need)
            if need > s._enc_end:                              # past the end of the stream: zero, under the pad mask
                s._feat = torch.cat([s._feat, torch.zeros(need - s._enc_end, C, device=dev)])
                s._enc_end = need
            tf, tm = s._text_at(self.L)
            for k in range(w.ka, w.kb):
                feats.append(s._feat[k * H - s._feat0:k * H - s._feat0 + W])
                texts.append(tf)
                masks.append(tm)
                pad = torch.ones(W, dtype=torch.bool, device=dev)
                align = torch.zeros(W, dtype=torch.long, device=dev)
                if n_valid is not None:
                    v = max(0, n_valid - k * H)
                    pad[v:] = False
                    align[v:] = 1                              # the processor's <pad> alignment for pad frames
                pads.append(pad)
                aligns.append(align)
                noise.append(stream_noise(s.seed, k * H, k * H + W, H, C, dev))
        n = len(feats)
        pick = lambda xs: torch.stack([xs[i] for i in slots])   # noqa: E731
        nb = len(slots)
        self.model._install_conditioning(pick(feats), pick(texts), pick(masks), None, self._ids.expand(nb, -1),
                                         pick(aligns), pick(pads), candidates=1)
        rows = pick(noise)
        self.model._ensure_engine().solve(rows, self.n_steps, rows, self.method)
        return rows[:n], job_windows

    def _blend(self, grp, rows: torch.Tensor):
        """Blend each stream's frames that became final from its previous window and the windows just solved; streams
        that finalise the same number of frames share one sab_blend_windows call (one output sequence each)."""
        W, H, C, dev = self.W, self.H, self.C, self.device
        by_count = defaultdict(list)
        i = 0
        for w in grp:
            s = w.key
            f_new = stream_final_frames(w.kb, W, s.n_final if s._ends_at(w.kb) else -1)
            by_count[f_new - s.final_frames].append((w, rows[i:i + w.kb - w.ka], f_new))
            i += w.kb - w.ka
        for count, members in by_count.items():
            wins, seq, start, flags = [], [], [], []
            for q, (w, solved, _) in enumerate(members):
                s = w.key
                last_group = s._ends_at(w.kb)
                ks = list(range(w.ka - (s._prev is not None), w.kb))
                if s._prev is not None:
                    wins.append(s._prev[None])
                wins.append(solved)
                seq += [q] * len(ks)
                start += [k * H - s.final_frames for k in ks]
                flags += [_capi.WIN_FIRST * (k == 0) + _capi.WIN_LAST * (last_group and k == w.kb - 1) for k in ks]
            win = torch.cat(wins).contiguous()
            out = torch.empty(len(members), count, C, device=dev, dtype=torch.float32)
            _capi.blend_windows(win, torch.tensor(seq, dtype=torch.int32, device=dev),
                                torch.tensor(start, dtype=torch.int32, device=dev),
                                torch.tensor(flags, dtype=torch.uint8, device=dev), self.O, out)
            for q, (w, solved, f_new) in enumerate(members):
                s = w.key
                s._lat = torch.cat([s._lat, out[q]])
                s.final_frames = f_new
                s.windows_solved = w.kb
                s._prev = solved[-1].clone()
                # the next window reads features from frame kb * H on
                drop = min(w.kb * H, s._enc_end) - s._feat0
                s._feat = s._feat[drop:].clone()
                s._feat0 += drop

    def _decode(self, grp, flushed: bool, jobs=(), drain: bool = False):
        """Decode frames [emitted_frames, emit_end) of each stream of the group from its final latent with halo_dec
        frames on each side; slices of equal length share one sab_decode.  Yields (stream, [2, samples]).  Jobs' tiles
        fill the call of steady slices, and their kept samples go to the job's output."""
        hop, halo = self.hop, self.halo_dec
        items = []                              # (stream, latent rows, first kept sample, end sample, job output offset)
        for w in grp:
            s = w.key
            a, F = s.emitted_frames, s.final_frames
            fl = s._ends_at(w.kb)
            b = stream_emit_end(F, halo, fl)
            if b <= a:
                items.append((s, None, 0, 0, None))
                continue
            d0, d1 = max(0, a - halo), F if fl else b + halo
            items.append((s, s._lat[d0 - s._lat0:d1 - s._lat0], (a - d0) * hop, (b - d0) * hop, None))
            s.emitted_frames = b
            keep0 = max(0, b - halo)                               # the next decode reads from here on
            s._lat = s._lat[keep0 - s._lat0:].clone()
            s._lat0 = keep0
        by_len = defaultdict(list)
        for i, j in enumerate(items):
            if j[1] is not None:
                by_len[j[1].shape[0]].append(i)
        steady = self._steady[1]
        if drain:
            by_len.setdefault(steady, [])                      # a drain tick has no live items: make the steady call
        wavs = {}
        eng = self.model._ensure_engine()
        for T, idx in by_len.items():
            if T == steady and (jobs or drain):
                slots, taken = self._call_slots(len(idx), flushed, False, jobs, SeparationJob._decode_offer, drain)
                if slots is None:
                    continue
                for j, t in zip(jobs, taken):
                    if not t:
                        continue
                    for start, k0, k1 in j._dec_tiles[j._dec_next:j._dec_next + t]:
                        idx.append(len(items))
                        items.append((j, j._lat[start - j._lat0:start - j._lat0 + T], (k0 - start) * hop,
                                      (k1 - start) * hop, k0 * hop))
                    j._dec_next += t
                    # the next tile reads from its start on (the last, right-aligned, may start before this one's end)
                    keep0 = j._dec_tiles[j._dec_next][0] if j._dec_next < len(j._dec_tiles) else j.final_frames
                    j._lat = j._lat[keep0 - j._lat0:].clone()
                    j._lat0 = keep0
            else:
                slots = self._slots(len(idx), flushed, solve=False)
            lat = torch.stack([items[idx[i]][1] for i in slots])
            out = torch.empty(len(slots), 2, T * hop, device=self.device, dtype=torch.float32)
            eng.decode(lat, len(slots), T, out)
            for i, ji in enumerate(idx):
                wavs[ji] = out[i]
        for i, (s, _, a, b, dst) in enumerate(items):
            if dst is not None:
                s._out[:, dst:dst + b - a].copy_(wavs[i][:, a:b])
            else:
                yield s, (torch.empty(2, 0, device=self.device) if i not in wavs else wavs[i][:, a:b])

    def _finish_jobs(self, jobs):
        """The jobs whose last tile has been decoded: their output at their own rate (one sab_resample call for all of
        them), then their state is released and they leave the queue."""
        sr = self.model.sample_rate
        done = [j for j in jobs if not j.done and j._dec_next == len(j._dec_tiles)]
        spread, ys = [], []                                     # keep_channels: the stems of every channel first
        for j in done:
            y = j._out
            if j.keep_channels:
                C, n, S = j._x48.shape[0], y.shape[1], j._x48.shape[1]
                y = torch.empty(2 * C, n, device=self.device, dtype=torch.float32)
                spread.append(dict(channels=C, target=j._out[0].data_ptr(), residual=j._out[1].data_ptr(), tr_first=0,
                                   tr_count=n, tr_length=n, mix=j._x48.data_ptr(), mix_channel_stride=S, mix_first=0,
                                   mix_count=S, mix_length=S, out_target=y[:C].data_ptr(),
                                   out_residual=y[C:].data_ptr(), out_channel_stride=n, out_first=0, out_count=n))
            ys.append(y)
        self.model._ensure_engine().spread_channels(spread)
        segs, outs = [], []
        for j, x in zip(done, ys):
            y = x
            if j.sample_rate != sr:
                n = x.shape[1]
                y = torch.empty(x.shape[0], resampled_length(n, sr, j.sample_rate), device=self.device,
                                dtype=torch.float32)
                segs += [dict(orig_rate=sr, new_rate=j.sample_rate, in_=x[r].data_ptr(), in_first=0, in_count=n,
                              length=n, out=y[r].data_ptr(), out_first=0, out_count=y.shape[1]) for r in range(x.shape[0])]
            outs.append(y)
        self.model._ensure_engine().resample(segs)
        for j, y in zip(done, outs):
            j._release()
            h = y.shape[0] // 2
            j._result = StreamOutput(target=y[:h] if j.keep_channels else y[0],
                                     residual=y[h:] if j.keep_channels else y[1])
            j.done = True
            self._jobs.remove(j)


def check_keep_channels(keep_channels) -> bool:
    if not isinstance(keep_channels, bool):
        raise TypeError(f"keep_channels must be True or False, got {keep_channels!r}")
    return keep_channels


def _drop_group(hold_plan_limits, key, jobs):
    """Finalizer of a stream group collected without close(): cancel its jobs and give back its plan residency."""
    for j in list(jobs):
        j.cancel()
    hold_plan_limits(key, None)
