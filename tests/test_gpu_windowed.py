"""GPU (H100) tests of recordings longer than the model's position table: the window cross-fade kernel
(blend_windows.cuh) through sab_blend_windows, and the windowed separate() built on it.

The tiny model with a short table (max_positions = 320, i.e. 12.8 s; rope_theta = max(10000, 640) = 10 000) makes 30-60 s
clips take 3-6 windows.  Bars as in test_gpu_longform.py: latent rel-L2 <= 5e-2,
cosine >= 0.998, waveform SNR >= 30 dB against the oracle; the kernel within 1e-6 of the fp64 blend.
"""
import pytest
import torch

from _util import rel_l2, snr_db

pytestmark = pytest.mark.gpu

TW = 320


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    assert torch.cuda.is_available()
    return _capi


@pytest.fixture(scope="module")
def short_cfg():
    from sam_audio_b200.config import stand_in_config
    cfg = stand_in_config("sam-audio-tiny", transformer={"max_positions": TW})
    assert cfg.transformer.rope_theta == 10000.0
    return cfg


@pytest.fixture(scope="module")
def short_model(capi, short_cfg, tiny_sd):
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    m = SAMAudio(short_cfg, text_encoder=SyntheticTextEncoder(short_cfg.text_encoder.dim))
    m.load_state_dict(tiny_sd)
    return m.eval().cuda()


def _blend_args(wins, c):
    from sam_audio_b200 import _capi
    seq = torch.tensor([w.clip * c + k for w in wins for k in range(c)], dtype=torch.int32, device="cuda")
    start = torch.tensor([w.start for w in wins for _ in range(c)], dtype=torch.int32, device="cuda")
    flags = torch.tensor([_capi.WIN_FIRST * w.first + _capi.WIN_LAST * w.last for w in wins for _ in range(c)],
                         dtype=torch.uint8, device="cuda")
    return seq, start, flags


def _rel_max(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max())


# ---------------------------------------------------------------------------------------------------------------
# the blend kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [1, 2])
@pytest.mark.parametrize("sizes,T", [([750, 250, 601], 750), ([1500], 1502), ([321, 900, 1], 901)])
def test_blend_reconstructs_and_matches_fp64(capi, sizes, T, c):
    """Several clips, c = 1 and 2: windows cut from one latent blend back to it, random windows match the fp64 blend,
    the NaN-prefilled output is finite everywhere, and frames no window covers (past each clip's end, or past Tw for a
    one-window clip) are exactly 0."""
    from _oracle_windowed import blend_fp64
    from sam_audio_b200.windows import window_layout, window_ramp
    wins = window_layout(sizes, TW)
    B, ramp = len(sizes), window_ramp(TW)
    g = torch.Generator(device="cuda").manual_seed(T + c)
    lat = torch.randn(B * c, T, 256, device="cuda", generator=g)
    seq, start, flags = _blend_args(wins, c)
    cut = torch.stack([lat[w.clip * c + k, w.start:w.start + TW] for w in wins for k in range(c)]).contiguous()
    out = torch.full_like(lat, float("nan"))
    capi.blend_windows(cut, seq, start, flags, ramp, out)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    for b, n in enumerate(sizes):
        rows, end = slice(b * c, (b + 1) * c), max(n, TW)
        assert _rel_max(out[rows, :end], lat[rows, :end]) < 1e-6
        assert bool((out[rows, end:] == 0).all())
    rnd = torch.randn(cut.shape, device="cuda", generator=g)
    out.fill_(float("nan"))
    capi.blend_windows(rnd, seq, start, flags, ramp, out)
    ref = blend_fp64(rnd.cpu(), wins, c, B, T, ramp)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert _rel_max(out.cpu(), ref) < 1e-6
    assert bool((out.cpu()[ref == 0] == 0).all())


# ---------------------------------------------------------------------------------------------------------------
# windowed separate()
# ---------------------------------------------------------------------------------------------------------------
def _batch(seconds, desc, anchors=None, seeds=None):
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip
    proc = SAMAudioProcessor(1920, 48000)
    auds = [synthetic_clip(s, int(48000 * sec)) for s, sec in zip(seeds or range(len(seconds)), seconds)]
    kw = {} if anchors is None else {"anchors": anchors}
    return lambda: proc(descriptions=desc, audios=auds, **kw)


def test_windowed_latent_is_the_blend_of_the_windows_solved_as_a_batch(short_model, capi):
    """The windowed path equals the composition done by hand: the windows of a 30 s and a 10 s clip cut out of the
    clips' inputs, installed as one batch through the ordinary prepare / solve, and blended."""
    from sam_audio_b200.synthetic import synthetic_descriptions, synthetic_noise
    from sam_audio_b200.windows import window_layout, window_ramp
    desc = synthetic_descriptions(2)
    make = _batch([30, 10], desc)
    noise = synthetic_noise(2, 750).cuda()
    short_model.separate(make().to("cuda"), noise=noise)
    got = short_model._last_latent.clone()

    m = short_model
    batch = make().to("cuda")
    feats = m._get_audio_features(batch.audios)
    tf, tm = m.text_encoder(batch.descriptions)
    wins = window_layout(batch.sizes, TW)
    assert [w.clip for w in wins] == [0, 0, 0, 1]
    sl = [slice(w.start, w.start + TW) for w in wins]
    m._install_conditioning(torch.stack([feats[w.clip, s] for w, s in zip(wins, sl)]),
                            torch.stack([tf[w.clip] for w in wins]), torch.stack([tm[w.clip] for w in wins]), None,
                            torch.stack([batch.anchor_ids[w.clip] for w in wins]),
                            torch.stack([batch.anchor_alignment[w.clip, s] for w, s in zip(wins, sl)]),
                            torch.stack([batch.audio_pad_mask[w.clip, s] for w, s in zip(wins, sl)]))
    y = torch.stack([noise[w.clip, s] for w, s in zip(wins, sl)]).contiguous()
    with torch.cuda.device(0):
        m._ensure_engine().solve(y, 16, y, "midpoint")
    want = torch.full_like(got, float("nan"))
    capi.blend_windows(y, *_blend_args(wins, 1), window_ramp(TW), want)
    torch.cuda.synchronize()
    assert torch.equal(got, want)


def test_grouping_does_not_change_the_result(short_model, monkeypatch):
    """One window per group (SAB_WINDOW_ROWS=1) against the default budget (all windows in one group): latent and both
    waveforms bit-equal."""
    from sam_audio_b200.synthetic import synthetic_descriptions, synthetic_noise
    desc = synthetic_descriptions(2)
    make = _batch([45, 20], desc, seeds=[3, 4])
    noise = synthetic_noise(2, 1125).cuda()
    a = short_model.separate(make().to("cuda"), noise=noise)
    la = short_model._last_latent.clone()
    monkeypatch.setenv("SAB_WINDOW_ROWS", "1")
    b = short_model.separate(make().to("cuda"), noise=noise)
    torch.cuda.synchronize()
    assert torch.equal(la, short_model._last_latent)
    for i in range(2):
        assert torch.equal(a.target[i], b.target[i]) and torch.equal(a.residual[i], b.residual[i])


def test_windowed_separate_vs_oracle(short_model, short_cfg, tiny_sd):
    """A 30 s clip (3 windows) whose anchor straddles the first window seam, batched with a 10 s clip (one padded
    window), against the oracle composed from the restated pieces."""
    from _oracle_windowed import separate_windowed
    from sam_audio_b200.synthetic import synthetic_noise, synthetic_text_features
    from sam_audio_b200.windows import window_layout, window_ramp
    desc = ["dog barking", "rain"]
    make = _batch([30, 10], desc, anchors=[[["+", 7.0, 14.5]], []], seeds=[7, 8])
    host = make()
    wins = window_layout(host.sizes, TW)
    assert wins[1].start * 1920 / 48000 < 14.5 and wins[0].start + TW > 7.0 * 25       # the anchor spans the seam
    noise = synthetic_noise(2, 750)
    out = short_model.separate(make().to("cuda"), noise=noise.cuda())
    lat = short_model._last_latent.cpu()
    tf, tm = synthetic_text_features(desc)
    tgt, res, ref_lat = separate_windowed(tiny_sd, short_cfg, host.audios, host.audio_pad_mask, host.sizes, tf, tm,
                                          host.anchor_ids, host.anchor_alignment, noise, wins, TW, window_ramp(TW),
                                          return_latent=True)
    cos = float(torch.nn.functional.cosine_similarity(lat.flatten().double(), ref_lat.flatten().double(), dim=0))
    assert rel_l2(lat, ref_lat) < 5e-2 and cos > 0.998
    for i in range(2):
        assert out.target[i].shape == tgt[i].shape
        assert snr_db(out.target[i].cpu(), tgt[i]) > 30.0 and snr_db(out.residual[i].cpu(), res[i]) > 30.0


def test_nothing_changes_at_or_below_the_table(short_model, capi, tiny_sd):
    """A 12 s clip (300 frames) takes the ordinary path below the table (320) and exactly at it (a model whose table
    ends at 300): bit-equal.  Both tables have rope_theta = 10 000 (max(10000, 2 * max_positions)); the default tiny
    config's 10 000-position table has rope_theta = 20 000, a different model, so it is not the comparison here."""
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.synthetic import synthetic_descriptions, synthetic_noise
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    cfg = stand_in_config("sam-audio-tiny", transformer={"max_positions": 300})
    assert cfg.transformer.rope_theta == 10000.0
    at = SAMAudio(cfg, text_encoder=SyntheticTextEncoder(cfg.text_encoder.dim))
    at.load_state_dict(tiny_sd)
    at = at.eval().cuda()
    make = _batch([12], synthetic_descriptions(1))
    assert int(make().sizes.max()) == 300
    noise = synthetic_noise(1, 300).cuda()
    a = short_model.separate(make().to("cuda"), noise=noise)
    b = at.separate(make().to("cuda"), noise=noise)
    assert torch.equal(short_model._last_latent, at._last_latent)
    assert torch.equal(a.target[0], b.target[0]) and torch.equal(a.residual[0], b.residual[0])


def test_past_the_old_ceiling(tiny_model):
    """The default tiny config (10 000 positions) on a 7 min clip (10 500 frames, 2 windows): the library raises no
    error, lengths are sizes x hop, outputs are finite, two runs are bit-equal."""
    from sam_audio_b200.synthetic import synthetic_noise
    from sam_audio_b200.windows import window_layout
    make = _batch([420], ["thunder"], seeds=[5])
    host = make()
    frames = int(host.sizes.max())
    assert frames == 10500 and len(window_layout(host.sizes, 10000)) == 2
    noise = synthetic_noise(1, frames).cuda()
    a = tiny_model.separate(make().to("cuda"), noise=noise)
    b = tiny_model.separate(make().to("cuda"), noise=noise)
    torch.cuda.synchronize()
    assert a.target[0].shape == (frames * 1920,) and a.residual[0].shape == (frames * 1920,)
    assert torch.isfinite(a.target[0]).all() and torch.isfinite(a.residual[0]).all()
    assert torch.equal(a.target[0], b.target[0]) and torch.equal(a.residual[0], b.residual[0])


def test_candidates_equal_the_single_candidate_run(short_model):
    """reranking_candidates = 2 with duplicated noise rows: each clip's result equals the single-candidate run."""
    from sam_audio_b200.synthetic import synthetic_descriptions, synthetic_noise
    desc = synthetic_descriptions(2)
    make = _batch([12, 30], desc)
    noise = synthetic_noise(2, 750).cuda()
    one = short_model.separate(make().to("cuda"), noise=noise)
    two = short_model.separate(make().to("cuda"), noise=noise.repeat_interleave(2, 0), reranking_candidates=2)
    for i in range(2):
        assert torch.equal(one.target[i], two.target[i]) and torch.equal(one.residual[i], two.residual[i])
