"""GPU (H100): visual-prompting front end — the frame pre-processing kernels (sab_preprocess_frames) against the oracle
restatement (pinned to torchvision, tests/test_oracle_vision.py), the PerceptionEncoder mirror's chunked encode against the
golden output of the reference's own class, and config-5-style separate() with masked video through a stand-in tower."""
import os

import pytest
import torch

from _util import rel_l2, snr_db

pytestmark = pytest.mark.gpu


def _levels(x):
    return ((x * 0.5 + 0.5) * 255).round()


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    return _capi


@pytest.mark.parametrize("shape", [(3, 3, 36, 64), (2, 3, 360, 640), (1, 3, 500, 300), (2, 3, 336, 336), (1, 3, 1080, 1920),
                                   (5, 3, 7, 5)])
def test_preprocess_frames_vs_oracle(capi, shape):
    from oracle import restate
    v = torch.randint(0, 256, shape, generator=torch.Generator().manual_seed(sum(shape)), dtype=torch.uint8)
    ours = capi.preprocess_frames(v.cuda(), 336).cpu()
    ref = restate.frame_transform(v)
    la, lb = _levels(ours), _levels(ref)
    assert ours.shape == ref.shape and float((la - lb).abs().max()) <= 1
    assert float((la != lb).float().mean()) < 1e-4            # same fp32 arithmetic: in practice identical
    assert torch.equal(ours[la == lb], ref[la == lb])
    assert float(ours.min()) >= -1.0 and float(ours.max()) <= 1.0


def test_perception_encoder_chunks_and_padding_vs_reference_golden(capi, golden_dir):
    """VisionEncoder.forward control flow (vision_encoder.py:47-69): 310 frames -> chunks of 300 + 10, pad_sequence zeros;
    golden = the reference's own PerceptionEncoder with the same stand-in tower."""
    from oracle.make_golden import FakeClip
    from sam_audio_b200.config import PerceptionEncoderConfig
    from sam_audio_b200.vision_encoder import PerceptionEncoder
    g = torch.load(os.path.join(golden_dir, "vision.pt"))
    gen = torch.Generator().manual_seed(g["seed"])
    vids = [torch.randint(0, 256, (n, 3, 20, 28), generator=gen, dtype=torch.uint8) for n in g["video_lens"]]
    big = torch.randint(0, 256, (2, 3, 360, 640), generator=gen, dtype=torch.uint8)
    calls = []

    class Tower(FakeClip):
        def encode_image(self, x, normalize=True):
            calls.append(x.shape[0])
            return super().encode_image(x, normalize)
    enc = PerceptionEncoder(PerceptionEncoderConfig(dim=FakeClip.DIM), model=Tower())
    out = enc([v.cuda() for v in vids]).cpu()
    assert calls == [300, 10, 7, 1]
    assert out.shape == g["feats"].shape and rel_l2(out, g["feats"]) < 1e-3
    assert float(out[1, 7:].abs().max()) == 0.0
    lv = _levels(enc.transform(big.cuda()).cpu()).to(torch.uint8)
    assert float((lv != g["big_levels"]).float().mean()) < 1e-4          # vs the reference's torchvision transform
    with pytest.raises(NotImplementedError):
        PerceptionEncoder(PerceptionEncoderConfig())([v.cuda() for v in vids])   # no tower attached: fails loudly


def test_separate_with_masked_video_vs_oracle(tiny_model, tiny_cfg, tiny_sd):
    """BASELINE config 5's path at test size: masked video frames -> PerceptionEncoder (native pre-processing + stand-in
    tower of the configured width) -> AlignModalities conditioning -> separate(), vs the oracle on the same features."""
    from oracle import restate
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import (synthetic_clip, synthetic_descriptions, synthetic_noise,
                                          synthetic_text_features)
    from sam_audio_b200.vision_encoder import PerceptionEncoder

    class Tower:
        def __init__(self, dim):
            self.proj = torch.randn(3 * 8 * 8, dim, generator=torch.Generator().manual_seed(9)) / 10.0

        def encode_image(self, x, normalize=True):
            f = torch.nn.functional.adaptive_avg_pool2d(x.float(), 8).flatten(1) @ self.proj.to(x.device)
            return torch.nn.functional.normalize(f, dim=-1) if normalize else f
    tower = Tower(tiny_cfg.vision_encoder.dim)
    proc = SAMAudioProcessor(1920, 48000)
    lens = [9600, 5000]
    auds = [synthetic_clip(40 + i, n) for i, n in enumerate(lens)]
    desc = synthetic_descriptions(2)
    gen = torch.Generator().manual_seed(3)
    vids = [torch.randint(0, 256, (9, 3, 24, 32), generator=gen, dtype=torch.uint8) for _ in lens]
    masks = [torch.randint(0, 2, (9, 1, 24, 32), generator=gen, dtype=torch.uint8) for _ in lens]
    masked = proc.mask_videos(vids, masks)
    host = proc(descriptions=desc, audios=auds, masked_videos=masked)
    noise = synthetic_noise(2, int(host.sizes.max()))
    prev = tiny_model.vision_encoder                  # the wrapper without a tower: visual prompting must fail loudly
    with pytest.raises(NotImplementedError):
        tiny_model.separate(proc(descriptions=desc, audios=auds, masked_videos=masked).to("cuda"), noise=noise.cuda())
    tiny_model.vision_encoder = PerceptionEncoder(tiny_cfg.vision_encoder, model=tower).cuda()
    try:
        out = tiny_model.separate(proc(descriptions=desc, audios=auds, masked_videos=masked).to("cuda"), noise=noise.cuda())
    finally:
        tiny_model.vision_encoder = prev
    vfeat = restate.vision_encode(host.masked_video, lambda x: tower.encode_image(x, True), tiny_cfg.vision_encoder.image_size,
                                  tiny_cfg.vision_encoder.batch_size).transpose(1, 2)           # [B, dim, T]
    tf, tm = synthetic_text_features(desc)
    tgt, res = restate.separate(tiny_sd, tiny_cfg, host.audios, host.audio_pad_mask, host.sizes, tf, tm, host.anchor_ids,
                                host.anchor_alignment, noise, video_features=vfeat)
    for ours, ref in zip(list(out.target) + list(out.residual), tgt + res):
        assert ours.shape == ref.shape and snr_db(ours.cpu(), ref) > 30.0
    # and it is not the text-only result
    plain = tiny_model.separate(proc(descriptions=desc, audios=auds).to("cuda"), noise=noise.cuda())
    assert snr_db(plain.target[0].cpu(), tgt[0]) < 25.0
