"""GPU (H100) tests of streaming separation (SAMAudio.stream, sam_audio_b200/stream.py): the output does not depend on
how the input is chunked, equals the offline composition of the same windows bit for bit, meets the oracle bar, and
holds bounded device memory."""
import math
import random

import pytest
import torch

from _util import snr_db

pytestmark = pytest.mark.gpu

HOP = 1920
DESC = "dog barking"


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as g
    g.build()
    assert torch.cuda.is_available()


@pytest.fixture(scope="module")
def small_model(built):
    from sam_audio_b200.model import build_synthetic_model
    return build_synthetic_model("sam-audio-small", seed=0, device="cuda:0", weights_device="cuda:0")


def _recording(seconds, extra=0, seed=11):
    from sam_audio_b200.synthetic import synthetic_clip
    return synthetic_clip(seed, int(48000 * seconds) + extra).reshape(-1).cuda()


def _run(model, wav, sizes, window_seconds=10.0, seed=0):
    """Push wav in chunks of the given sizes (the rest, if any, in one last chunk), flush; returns (target, residual)
    concatenated over every call."""
    s = model.stream(DESC, window_seconds=window_seconds, seed=seed)
    outs, i = [], 0
    for n in sizes:
        if i >= wav.numel():
            break
        outs.append(s.push(wav[i:i + n]))
        i += n
    if i < wav.numel():
        outs.append(s.push(wav[i:]))
    outs.append(s.flush())
    torch.cuda.synchronize()
    return torch.cat([o.target for o in outs]), torch.cat([o.residual for o in outs])


def _random_sizes(n, seed):
    rng = random.Random(seed)
    sizes, total = [], 0
    while total < n:
        s = rng.choice([1, 1, 7, 1919, 1921, 4801, 30_000, 96_001, 500_000])
        sizes.append(s)
        total += s
    return sizes


def _offline(model, wav, W, seed=0):
    """The offline composition of the stream's windows: whole-recording encode, SAMAudio._solve_windows on
    stream_window_starts(T, W) with the stream's noise (features zero and masked past T), whole-recording decode."""
    from sam_audio_b200.stream import stream_noise
    from sam_audio_b200.windows import Window, stream_hop, stream_window_starts
    m = model
    with torch.cuda.device(0):
        feats = m._get_audio_features(wav.view(1, 1, -1))
        T = feats.shape[1]
        starts = stream_window_starts(T, W)
        Te = starts[-1] + W
        fe = torch.zeros(1, Te, 256, device="cuda")
        fe[:, :T] = feats
        pad = torch.zeros(1, Te, dtype=torch.bool, device="cuda")
        pad[:, :T] = True
        align = torch.ones(1, Te, dtype=torch.long, device="cuda")
        align[:, :T] = 0
        ids = torch.tensor([[0, 3]], dtype=torch.long, device="cuda")
        tf, tm = m.text_encoder([DESC])
        noise = stream_noise(seed, 0, Te, stream_hop(W), device="cuda")[None].contiguous()
        wins = [Window(0, s, i == 0, i == len(starts) - 1) for i, s in enumerate(starts)]
        lat = m._solve_windows(fe, tf, tm, None, ids, align, pad, wins, W, noise, 1, 16, "midpoint")
        wavs = torch.empty(1, 2, T * HOP, device="cuda")
        m._ensure_engine().decode(lat[:, :T].contiguous(), 1, T, wavs)
    torch.cuda.synchronize()
    return wavs[0, 0], wavs[0, 1]


@pytest.fixture(scope="module")
def long_wav():
    return _recording(75, extra=1234)           # 1875 frames + a partial one (reflect-padded at flush)


@pytest.fixture(scope="module")
def tiny_one_chunk(tiny_model, long_wav):
    return _run(tiny_model, long_wav, [long_wav.numel()])


def test_chunking_does_not_change_a_bit(tiny_model, long_wav, tiny_one_chunk):
    """75 s at the default 10 s windows (9 windows): one chunk, 4 800-sample chunks, random chunk sizes (1-sample chunks,
    sizes that are not multiples of the hop), and nearly everything in the last push before flush(): bit-identical
    target and residual, ceil(n / hop) * hop samples each."""
    n = long_wav.numel()
    tgt, res = tiny_one_chunk
    assert tgt.shape == res.shape == (math.ceil(n / HOP) * HOP,)
    assert torch.isfinite(tgt).all() and torch.isfinite(res).all()
    for sizes in ([4800] * (n // 4800 + 1), _random_sizes(n, 0), _random_sizes(n, 1), [1, 2, n - 4, 1]):
        t, r = _run(tiny_model, long_wav, sizes)
        assert torch.equal(t, tgt) and torch.equal(r, res)


def test_chunking_on_the_small_stand_in(small_model):
    """The same on the sam-audio-small stand-in with 2 s windows (W = 50) over 20 s."""
    wav = _recording(20, extra=77, seed=5)
    tgt, res = _run(small_model, wav, [wav.numel()], window_seconds=2.0)
    for sizes in ([48000] * 21, _random_sizes(wav.numel(), 2)):
        t, r = _run(small_model, wav, sizes, window_seconds=2.0)
        assert torch.equal(t, tgt) and torch.equal(r, res)


def test_equals_the_offline_composition(tiny_model, long_wav, tiny_one_chunk):
    """The stream's output equals, bit for bit, the whole-recording encode, the windows of stream_window_starts solved
    by SAMAudio._solve_windows from the same noise, and the whole-recording decode."""
    t, r = _offline(tiny_model, long_wav, 250)
    assert torch.equal(t, tiny_one_chunk[0]) and torch.equal(r, tiny_one_chunk[1])


def test_equals_the_offline_composition_short_windows(small_model):
    wav = _recording(20, extra=77, seed=5)
    t, r = _offline(small_model, wav, 50)
    st, sr = _run(small_model, wav, [48000] * 21, window_seconds=2.0)
    assert torch.equal(t, st) and torch.equal(r, sr)


@pytest.fixture(scope="module")
def oracle_stream(tiny_cfg, tiny_sd):
    """The stream composed from the restated pieces of oracle/restate.py, as tests/_oracle_windowed.py composes
    separate(): codec encode of the whole recording (reflect-padded), the midpoint solve of every window of
    stream_window_starts on its slice (features zero and masked past the end), the fp64 blend, codec decode."""
    from _oracle_windowed import blend_fp64
    from oracle import restate
    from sam_audio_b200.stream import stream_noise
    from sam_audio_b200.synthetic import synthetic_text_features
    from sam_audio_b200.windows import Window, stream_hop, stream_window_starts, window_ramp
    cfg, sd = tiny_cfg, tiny_sd
    cc = cfg.audio_codec

    def run(wav, W, seed=0):
        feats = restate.codec_encode(sd, cc, wav.view(1, 1, -1)).transpose(1, 2)
        feats = torch.cat([feats, feats], 2)
        T = feats.shape[1]
        starts = stream_window_starts(T, W)
        Te = starts[-1] + W
        fe = torch.zeros(1, Te, 256)
        fe[:, :T] = feats
        pad = torch.arange(Te) < T
        align = (~pad).long()
        ids = torch.tensor([0, 3])
        tf, tm = synthetic_text_features([DESC])
        noise = stream_noise(seed, 0, Te, stream_hop(W), device="cuda").cpu()
        wins = [Window(0, s, i == 0, i == len(starts) - 1) for i, s in enumerate(starts)]
        lats = []
        for w in wins:
            sl = slice(w.start, w.start + W)
            fa = dict(audio_features=fe[:, sl], text_features=tf, text_mask=tm,
                      masked_video_features=torch.zeros(1, cfg.vision_encoder.dim, W), anchor_ids=ids[None],
                      anchor_alignment=align[None, sl], audio_pad_mask=pad[None, sl])

            def field(t, y):
                return restate.samaudio_forward(sd, cfg, y, time=t.expand(y.shape[0]), **fa)
            lats.append(restate.odeint_midpoint(field, noise[None, sl], 16))
        lat = blend_fp64(torch.cat(lats), wins, 1, 1, Te, window_ramp(W)).float()[:, :T]
        wavs = restate.codec_decode(sd, cc, lat.transpose(1, 2).reshape(2, cc.codebook_dim, T)).view(2, -1)
        return wavs[0], wavs[1]
    return run


@pytest.mark.parametrize("window_seconds", [2.0, 10.0])
def test_against_the_oracle(tiny_model, oracle_stream, window_seconds):
    """W = 50 (11 windows) and the default W = 250 (3 windows) over 20 s pushed in 1 s chunks: >= 30 dB wav SNR."""
    wav = _recording(20, extra=999, seed=9)
    tgt, res = _run(tiny_model, wav, [48000] * 21, window_seconds=window_seconds)
    ref_t, ref_r = oracle_stream(wav.cpu(), int(round(window_seconds * 25)))
    assert tgt.shape == ref_t.shape
    assert snr_db(tgt.cpu(), ref_t) > 30.0 and snr_db(res.cpu(), ref_r) > 30.0


def test_memory_is_bounded(tiny_model):
    """1 s pushes at W = 50: the engine's workspace and the allocator's peak after 20 windows equal those after 3."""
    wav = _recording(40, seed=3)
    s = tiny_model.stream(DESC, window_seconds=2.0)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    at = {}
    for i in range(0, wav.numel(), 48000):
        s.push(wav[i:i + 48000])
        if s.windows_solved in (3, 20) and s.windows_solved not in at:
            torch.cuda.synchronize()
            at[s.windows_solved] = (s.workspace_bytes(), torch.cuda.max_memory_allocated())
    s.flush()
    assert set(at) == {3, 20}
    assert at[20] == at[3]


def test_a_flushed_stream_is_closed(tiny_model):
    s = tiny_model.stream(DESC, window_seconds=2.0)
    out = s.push(_recording(1, seed=1))
    assert out.target.numel() == 0                       # no window is ready after 1 s of a 2 s window
    tail = s.flush()
    assert tail.target.shape == tail.residual.shape == (25 * HOP,)
    with pytest.raises(RuntimeError, match="closed"):
        s.push(torch.zeros(10, device="cuda"))
    with pytest.raises(RuntimeError, match="closed"):
        s.flush()
    assert tiny_model.stream(DESC).flush().target.numel() == 0
