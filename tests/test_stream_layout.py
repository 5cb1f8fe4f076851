"""CPU: the window layout of streams (sam_audio_b200.windows, stream_* functions), the stream's noise, and the argument
checks of SAMAudio.stream()."""
import math
import random

import pytest
import torch

from sam_audio_b200.windows import (stream_emit_end, stream_final_frames, stream_frames_available, stream_hop,
                                    stream_window_frames, stream_window_starts, stream_windows_ready, window_ramp)

HOP, HALO_ENC, HALO_DEC = 1920, 6, 8          # the standard codec rates (sab_codec_tiling reports these halos)
WS = [8, 9, 50, 64, 250, 256, 1000]


@pytest.mark.parametrize("W", WS)
def test_layout_is_prefix_stable(W):
    """The windows of a shorter stream are a prefix of a longer one's, and the windows ready before flush() at any
    sample count are a prefix of the final layout whatever the stream's final length."""
    full = stream_window_starts(20 * W, W)
    for n in range(1, 20 * W, max(1, W // 7)):
        assert full[:len(stream_window_starts(n, W))] == stream_window_starts(n, W)
    for n_samples in range(0, 20 * W * HOP, 7919):
        ready = stream_windows_ready(stream_frames_available(n_samples, HOP, HALO_ENC), W)
        for n_final in (math.ceil(n_samples / HOP), math.ceil(n_samples / HOP) + 1, 25 * W):
            if n_final:
                assert ready <= len(stream_window_starts(n_final, W))


@pytest.mark.parametrize("W", WS)
@pytest.mark.parametrize("n", [1, 7, 8, 9, 43, 44, 45, 50, 51, 95, 250, 251, 469, 470, 1875, 10007])
def test_layout_covers_with_exact_overlaps(n, W):
    H, O = stream_hop(W), window_ramp(W)
    assert O == W // 8 and H == W - O
    starts = stream_window_starts(n, W)
    assert starts == [k * H for k in range(len(starts))]
    assert starts[-1] < n and starts[-1] + W >= n                           # the last window covers the last frame
    assert len(starts) == 1 or starts[-2] + W < n                           # ... and is needed
    assert all(b - a == H and a + W - b == O for a, b in zip(starts, starts[1:]))
    covered = torch.zeros(n, dtype=torch.bool)
    for s in starts:
        covered[s:s + W] = True
    assert bool(covered.all())


@pytest.mark.parametrize("W", WS)
def test_ready_and_final_rules(W):
    H = stream_hop(W)
    for n in range(0, 6 * W):
        k = stream_windows_ready(n, W)
        assert all(j * H + W <= n for j in range(k)) and k * H + W > n       # exactly the windows inside [0, n)
    assert stream_frames_available(0, HOP, HALO_ENC) == 0
    assert stream_frames_available((W + HALO_ENC) * HOP, HOP, HALO_ENC) == W
    assert stream_frames_available((W + HALO_ENC) * HOP - 1, HOP, HALO_ENC) == W - 1
    for m in range(0, 12):
        F = stream_final_frames(m, W)
        for t in range(0, (m + 2) * H):
            covering = [j for j in range(t // H + 2) if j * H <= t < j * H + W]
            assert (t < F) == (max(covering) < m)                            # final = every covering window solved
    assert stream_final_frames(3, W, n_final=1234) == 1234
    assert stream_emit_end(100, HALO_DEC, False) == 92 and stream_emit_end(5, HALO_DEC, False) == 0
    assert stream_emit_end(100, HALO_DEC, True) == 100


def _schedule(pushes, W):
    """Host replay of a stream's schedule: after each push (and at flush), windows solved, final and emitted frames."""
    n, solved, emitted, events = 0, 0, 0, []
    for S in pushes:
        n += S
        solved = max(solved, stream_windows_ready(stream_frames_available(n, HOP, HALO_ENC), W))
        final = stream_final_frames(solved, W)
        e = max(emitted, stream_emit_end(final, HALO_DEC, False))
        events.append((n, solved, final, emitted, e, False))
        emitted = e
    T = math.ceil(n / HOP)
    solved = len(stream_window_starts(T, W))
    final = stream_final_frames(solved, W, n_final=T)
    events.append((n, solved, final, emitted, stream_emit_end(final, HALO_DEC, True), True))
    return T, events


@pytest.mark.parametrize("W", [8, 50, 250])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_emission_never_precedes_the_covering_windows(W, seed):
    """A frame is emitted only once every window that covers it is solved and frames up to it + the decoder halo are
    final; emission is contiguous and monotone; after flush() exactly ceil(n / hop) frames, ceil(n / hop) * hop
    samples, have been emitted."""
    rng = random.Random(seed)
    pushes = [rng.choice([1, 7, 1919, 1921, 4800, 48000, 250_000]) for _ in range(rng.randint(1, 120))]
    T, events = _schedule(pushes, W)
    starts = stream_window_starts(T, W)
    total = 0
    for n, solved, final, e0, e1, flushed in events:
        assert e1 >= e0
        assert solved <= len(starts)
        for t in range(e0, e1):
            assert all(k < solved for k, s in enumerate(starts) if s <= t < s + W)
            assert flushed or t + HALO_DEC < final
        total += e1 - e0
        if not flushed:
            assert solved == 0 or (solved - 1) * stream_hop(W) + W + HALO_ENC <= n // HOP   # encoder context arrived
    assert total == T and total * HOP == math.ceil(sum(pushes) / HOP) * HOP


def test_noise_is_a_function_of_seed_and_frame():
    from sam_audio_b200.stream import stream_noise
    whole = stream_noise(3, 0, 700, 219, device="cpu")
    assert whole.shape == (700, 256)
    for a, b in [(0, 250), (219, 469), (438, 688), (5, 6), (218, 220)]:
        assert torch.equal(stream_noise(3, a, b, 219, device="cpu"), whole[a:b])
    assert not torch.equal(stream_noise(4, 0, 700, 219, device="cpu"), whole)
    assert not torch.equal(whole[:219], whole[219:438])


@pytest.fixture(scope="module")
def cpu_model():
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    cfg = stand_in_config("sam-audio-tiny", transformer={"max_positions": 320})
    return SAMAudio(cfg, text_encoder=SyntheticTextEncoder(cfg.text_encoder.dim))


def test_window_length_is_checked(cpu_model):
    assert stream_window_frames(10.0, 25.0, 10000) == 250
    assert stream_window_frames(0.32, 25.0, 10000) == 8
    assert stream_window_frames(12.8, 25.0, 320) == 320
    for sec in (0.28, 0.0, -1.0, 12.84):
        with pytest.raises(ValueError, match="8 <= W <= 320"):
            cpu_model.stream("rain", window_seconds=sec)


@pytest.mark.parametrize("kw,why", [(dict(reranking_candidates=2), "rankers"),
                                    (dict(anchors=[["+", 1.0, 2.0]]), "time base"),
                                    (dict(masked_video=torch.zeros(4, 3, 8, 8)), "time base")])
def test_unsupported_prompts_are_refused(cpu_model, kw, why):
    with pytest.raises(NotImplementedError, match=why):
        cpu_model.stream("rain", window_seconds=10.0, **kw)


def test_ode_options_are_checked_as_in_separate(cpu_model):
    with pytest.raises(NotImplementedError, match="fixed-grid"):
        cpu_model.stream("rain", window_seconds=10.0, ode_opt={"method": "dopri5"})
