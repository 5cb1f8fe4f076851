"""GPU (H100) parity at the BENCHMARKED shapes — sam-audio-large (d 2816 / 22 heads / 24 layers) and sam-audio-small —
against the fp32 CPU oracle: one ODE function evaluation at T = 250 with ragged masks, the full 32-evaluation
separate() of a 10 s @ 48 kHz clip (error compounding at production depth x length), and batch invariance of a clip
inside the B = 64 batch bench.py times.

Tolerances (bf16 tensor-core operands, fp32 accumulation; the reference is fp32 end to end):
  one evaluation ........ rel-L2 <= 2e-2      latent after 32 evaluations ..... rel-L2 <= 5e-2, cosine >= 0.998
  waveforms ............. SNR >= 30 dB        batch invariance ................ >= 60 dB (bit-equal in practice)
"""
import pytest
import torch

from _util import rel_l2, snr_db

pytestmark = pytest.mark.gpu


def _model(name, seed):
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200.config import stand_in_config
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.synthetic import make_state_dict
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    cfg = stand_in_config(name)
    sd = make_state_dict(cfg, seed=seed)
    m = SAMAudio(cfg, text_encoder=SyntheticTextEncoder())
    m.load_state_dict(sd)
    m = m.eval().cuda()
    m._ensure_engine()
    m._state = None          # the engine holds the packed copy; the fp32 dict stays with the oracle only
    return m, cfg, sd


@pytest.fixture(scope="module")
def large():
    return _model("sam-audio-large", 2)


def _forward_vs_oracle(m, cfg, sd):
    from oracle import restate
    g = torch.Generator().manual_seed(17)
    B, T, L = 2, 250, 3
    noisy = torch.randn(B, T, 256, generator=g)
    f = torch.randn(B, T, 128, generator=g)
    feats = torch.cat([f, f], 2)
    text = torch.randn(B, L, 768, generator=g)
    tmask = torch.tensor([[True, True, True], [True, True, False]])
    pad = restate.mask_from_sizes(torch.tensor([250.0, 187.0]))
    ids, al = restate.process_anchors([[["+", 1.0, 3.0]], [["-", 0.5, 6.0]]], pad, 1920, 48000)
    time = torch.tensor([0.40625, 0.96875])
    ref = restate.samaudio_forward(sd, cfg, noisy, feats, text, time, torch.zeros(B, 1024, T), tmask, ids, al, pad)
    out = m.forward(noisy.cuda(), feats.cuda(), text.cuda(), time.cuda(), masked_video_features=torch.zeros(B, 1024, T).cuda(),
                    text_mask=tmask.cuda(), anchor_ids=ids.cuda(), anchor_alignment=al.cuda(), audio_pad_mask=pad.cuda())
    return rel_l2(out.cpu(), ref)


def _separate_vs_oracle(m, cfg, sd, clip_seed):
    from oracle import restate
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_noise, synthetic_text_features
    proc = SAMAudioProcessor(1920, 48000)
    aud, desc = [synthetic_clip(clip_seed)], ["dog barking"]
    host = proc(descriptions=desc, audios=aud)
    noise = synthetic_noise(1, 250)
    out = m.separate(proc(descriptions=desc, audios=aud).to("cuda"), noise=noise.cuda())     # 16 midpoint steps
    lat = m._last_latent.cpu()
    tf, tm = synthetic_text_features(desc)
    tgt, res, ref_lat = restate.separate(sd, cfg, host.audios, host.audio_pad_mask, host.sizes, tf, tm, host.anchor_ids,
                                         host.anchor_alignment, noise, return_latent=True)
    assert out.target[0].shape == (480000,)
    cos = float(torch.nn.functional.cosine_similarity(lat.flatten().double(), ref_lat.flatten().double(), dim=0))
    return dict(latent_rel_l2=rel_l2(lat, ref_lat), latent_cos=cos, snr_target=snr_db(out.target[0].cpu(), tgt[0]),
                snr_residual=snr_db(out.residual[0].cpu(), res[0]))


def test_large_one_evaluation_vs_oracle(large):
    """SAMAudio.forward at sam-audio-large (rmsnorm_mod_kernel<22>, QKV N = 8448, w13 N = 15104), B = 2, T = 250,
    ragged pad mask, ragged text mask, anchors."""
    e = _forward_vs_oracle(*large)
    print(f"\n[large] one evaluation rel-L2 {e:.3e}")
    assert e < 2e-2


def test_large_full_32_evaluations_vs_oracle(large):
    """The benchmarked model through the whole path: one 10 s clip, 16 midpoint steps = 32 evaluations, 24 layers."""
    r = _separate_vs_oracle(*large, clip_seed=5)
    print(f"\n[large] 32 evaluations: {r}")
    assert r["latent_rel_l2"] < 5e-2 and r["latent_cos"] > 0.998
    assert r["snr_target"] > 30.0 and r["snr_residual"] > 30.0


def test_large_batch_invariance_b64(large):
    """Clip 0 separated alone == clip 0 inside the B = 64 batch that bench.py times (every op is per sequence; the
    GEMM tiles, 2-CTA clusters and codec chunks it lands in differ)."""
    m = large[0]
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_descriptions, synthetic_noise
    proc = SAMAudioProcessor(1920, 48000)
    B = 64
    auds = [synthetic_clip(i) for i in range(B)]
    desc = synthetic_descriptions(B)
    noise = synthetic_noise(B, 250).cuda()
    full = m.separate(proc(descriptions=desc, audios=auds).to("cuda"), noise=noise)
    t0, r0 = full.target[0].clone(), full.residual[0].clone()
    t63 = full.target[63].clone()
    del full
    one = m.separate(proc(descriptions=desc[:1], audios=auds[:1]).to("cuda"), noise=noise[:1])
    last = m.separate(proc(descriptions=desc[63:], audios=auds[63:]).to("cuda"), noise=noise[63:])
    s = min(snr_db(t0, one.target[0]), snr_db(r0, one.residual[0]), snr_db(t63, last.target[0]))
    print(f"\n[large] B=64 vs alone: bit-equal={torch.equal(t0, one.target[0])}, worst SNR {s:.1f} dB")
    assert s > 60.0


def test_small_full_32_evaluations_vs_oracle():
    """sam-audio-small stand-in (BASELINE config 1's model), one 10 s clip, 32 evaluations."""
    m, cfg, sd = _model("sam-audio-small", 3)
    e = _forward_vs_oracle(m, cfg, sd)
    r = _separate_vs_oracle(m, cfg, sd, clip_seed=6)
    print(f"\n[small] one evaluation rel-L2 {e:.3e}; 32 evaluations: {r}")
    assert e < 2e-2
    assert r["latent_rel_l2"] < 5e-2 and r["latent_cos"] > 0.998
    assert r["snr_target"] > 30.0 and r["snr_residual"] > 30.0
