"""GPU (H100) tests of long clips (T > 256 latent frames, i.e. more than 10 s): the wgmma streaming self-attention
kernel (attention_stream_tc.cuh) through its C-ABI seam, and the DiT / separate() paths that use it, against fp32
torch, the mma.sync streaming kernel and the CPU oracle.

Tolerances as in test_gpu_parity.py / test_gpu_parity_large.py:
  attention vs fp32 softmax(QK^T)V on the same bf16 operands ...... rel-L2 <= 1e-2
  attention vs attention_kernel on the same inputs ................ rel-L2 <= 3e-3
  one DiT evaluation vs oracle .................................... rel-L2 <= 2e-2
  32 evaluations: latent rel-L2 <= 5e-2, cosine >= 0.998, waveforms SNR >= 30 dB
"""
import pytest
import torch

from _util import rel_l2, snr_db

pytestmark = pytest.mark.gpu

LOG2E = 1.4426950408889634
LN2 = 0.6931471805599453


@pytest.fixture(scope="module")
def capi():
    import __graft_entry__ as g
    g.build()
    from sam_audio_b200 import _capi
    assert torch.cuda.is_available()
    return _capi


def _ragged_mask(items, T):
    """Item 0's valid keys end inside the first 128-key block, item 1's whole last block is masked, the others lose
    a few keys at the end (item 2 none)."""
    mask = torch.ones(items, T, dtype=torch.uint8, device="cuda")
    last_block = 128 * ((T + 127) // 128 - 1)
    mask[0, 70:] = 0
    if items > 1:
        mask[1, last_block - 5:] = 0
    for i in range(3, items):
        mask[i, T - 3 * i:] = 0
    return mask


def _reference(q, k, v, mask, items, heads, T, scale):
    qf, kf, vf = (x.float().view(items, T, heads, 128).permute(0, 2, 1, 3) for x in (q, k, v))
    s = (qf @ kf.transpose(-1, -2) * scale).masked_fill(~mask.bool()[:, None, None, :], float("-inf"))
    return (torch.softmax(s, -1) @ vf).permute(0, 2, 1, 3).reshape(items * T, heads * 128), s


@pytest.mark.parametrize("exact", [False, True])
@pytest.mark.parametrize("items,heads,T", [(3, 2, 257), (4, 3, 300), (2, 2, 384), (5, 4, 750), (3, 4, 1500), (2, 3, 4097)])
def test_streaming_tc_attention_vs_torch(capi, items, heads, T, exact):
    """Every shape has several 128-query CTAs per (item, head) sharing that head's K / V stream; T covers one key
    past two blocks, a short last block, a whole number of blocks and more blocks than ring stages.  exact = online
    running maximum with rescale; otherwise the bounded variant, fed q already in the log2 domain as the engine's QKV
    epilogue leaves it.  Polynomial exp2 on 3 of 8 pairs or none.  The output starts as NaN: every row < T is written
    and no masked block leaks a NaN."""
    g = torch.Generator(device="cuda").manual_seed(T + items)
    q, k, v = (torch.randn(items * T, heads * 128, device="cuda", generator=g).bfloat16() for _ in range(3))
    mask = _ragged_mask(items, T)
    if exact:
        qin, shift = q, -1.0
        ref, _ = _reference(q, k, v, mask, items, heads, T, 1.0 / 128 ** 0.5)
    else:
        qin, shift = (q.float() * (LOG2E / 128 ** 0.5)).bfloat16(), 0.0
        ref, s = _reference(qin, k, v, mask, items, heads, T, LN2)
        assert float(s[torch.isfinite(s)].abs().max()) < 50 * LN2
        del s
    o = torch.empty(items * T, heads * 128, device="cuda", dtype=torch.bfloat16)
    for poly in (3, 0):
        o.fill_(float("nan"))
        capi.check(capi.lib().sab_test_attention_stream(items, heads, T, qin.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                        mask.data_ptr(), o.data_ptr(), shift, poly, capi.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.isfinite(o.float()).all()
        assert rel_l2(o.float(), ref) < 1e-2, (poly, exact)


@pytest.mark.parametrize("items,heads,T", [(3, 2, 300), (3, 4, 1500)])
def test_streaming_tc_attention_vs_mma_sync_kernel(capi, items, heads, T):
    """The two streaming kernels on the same inputs: both round P and the output to bf16, so they agree more closely
    with each other than either does with fp32."""
    g = torch.Generator(device="cuda").manual_seed(T)
    q, k, v = (torch.randn(items * T, heads * 128, device="cuda", generator=g).bfloat16() for _ in range(3))
    mask = _ragged_mask(items, T)
    a = torch.full((items * T, heads * 128), float("nan"), device="cuda", dtype=torch.bfloat16)
    b = torch.full_like(a, float("nan"))
    capi.check(capi.lib().sab_test_attention_stream(items, heads, T, q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                    mask.data_ptr(), a.data_ptr(), -1.0, 0, capi.stream_ptr()))
    capi.check(capi.lib().sab_test_attention(items, heads, T, T, q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                             mask.data_ptr(), b.data_ptr(), capi.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.isfinite(a.float()).all() and torch.isfinite(b.float()).all()
    assert rel_l2(a.float(), b.float()) < 3e-3


def test_streaming_tc_attention_without_mask(capi):
    """No key mask at all (null pointer): keys >= T of the last block are still excluded."""
    items, heads, T = 2, 2, 333
    g = torch.Generator(device="cuda").manual_seed(9)
    q, k, v = (torch.randn(items * T, heads * 128, device="cuda", generator=g).bfloat16() for _ in range(3))
    ones = torch.ones(items, T, dtype=torch.uint8, device="cuda")
    ref, _ = _reference(q, k, v, ones, items, heads, T, 1.0 / 128 ** 0.5)
    o = torch.full((items * T, heads * 128), float("nan"), device="cuda", dtype=torch.bfloat16)
    capi.check(capi.lib().sab_test_attention_stream(items, heads, T, q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                    None, o.data_ptr(), -1.0, 3, capi.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.isfinite(o.float()).all() and rel_l2(o.float(), ref) < 1e-2


# ---------------------------------------------------------------------------------------------------------------
# one DiT evaluation at T = 750 (30 s) against the oracle, through each self-attention path
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def long_eval(tiny_cfg, tiny_sd):
    from oracle import restate
    g = torch.Generator().manual_seed(750)
    B, T, L = 3, 750, 5
    noisy = torch.randn(B, T, 256, generator=g)
    f = torch.randn(B, T, 128, generator=g)
    feats = torch.cat([f, f], 2)
    text = torch.randn(B, L, 768, generator=g)
    tmask = torch.ones(B, L, dtype=torch.bool)
    tmask[1, 3:] = False
    pad = restate.mask_from_sizes(torch.tensor([750.0, 601.0, 100.0]))     # clip 2 ends inside the first key block
    ids, al = restate.process_anchors([[["+", 1.0, 23.0]], [["-", 0.5, 6.0], ["+", 11.0, 20.0]], []], pad, 1920, 48000)
    time = torch.tensor([0.40625, 0.96875, 0.0])
    ref = restate.samaudio_forward(tiny_sd, tiny_cfg, noisy, feats, text, time, torch.zeros(B, 1024, T), tmask, ids, al, pad)
    return dict(noisy=noisy, feats=feats, text=text, tmask=tmask, pad=pad, ids=ids, al=al, time=time, ref=ref)


@pytest.mark.parametrize("switch", [None, "SAB_ATTN_EXACT", "SAB_NO_TC_ATTENTION"])
def test_dit_evaluation_30s_vs_oracle(tiny_cfg, tiny_sd, long_eval, monkeypatch, switch):
    """Ragged pad masks, ragged text mask and anchors at T = 750.  The default engine runs the wgmma streaming kernel
    with whichever softmax the layers' logit bounds select, SAB_ATTN_EXACT forces its online-maximum variant and
    SAB_NO_TC_ATTENTION the mma.sync kernel: all three stay pinned to the oracle."""
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    if switch:
        monkeypatch.setenv(switch, "1")
    m = SAMAudio(tiny_cfg, text_encoder=SyntheticTextEncoder())
    m.load_state_dict(tiny_sd)
    m = m.eval().cuda()
    d = long_eval
    B, T = d["noisy"].shape[:2]
    out = m.forward(d["noisy"].cuda(), d["feats"].cuda(), d["text"].cuda(), d["time"].cuda(),
                    masked_video_features=torch.zeros(B, 1024, T).cuda(), text_mask=d["tmask"].cuda(),
                    anchor_ids=d["ids"].cuda(), anchor_alignment=d["al"].cuda(), audio_pad_mask=d["pad"].cuda())
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert rel_l2(out.cpu(), d["ref"]) < 2e-2


# ---------------------------------------------------------------------------------------------------------------
# separate() of long clips on the tiny model
# ---------------------------------------------------------------------------------------------------------------
def test_batch_invariance_30s_clip(tiny_model):
    """A 30 s clip separated alone == the same clip in a batch with a 10 s clip (every op is per sequence; the 10 s
    clip's keys past its length are whole masked blocks of the streaming kernel)."""
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_descriptions, synthetic_noise
    proc = SAMAudioProcessor(1920, 48000)
    auds = [synthetic_clip(0, 48000 * 30), synthetic_clip(1, 48000 * 10)]
    desc = synthetic_descriptions(2)
    noise = synthetic_noise(2, 750).cuda()
    both = tiny_model.separate(proc(descriptions=desc, audios=auds).to("cuda"), noise=noise)
    one = tiny_model.separate(proc(descriptions=desc[:1], audios=auds[:1]).to("cuda"), noise=noise[:1])
    assert both.target[0].shape == (48000 * 30,) and both.target[1].shape == (48000 * 10,)
    assert torch.equal(both.target[0], one.target[0]) and torch.equal(both.residual[0], one.residual[0])
    assert torch.isfinite(both.target[1]).all()


def test_separate_60s_clip_shape_finite_deterministic(tiny_model):
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_noise
    proc = SAMAudioProcessor(1920, 48000)
    n = 48000 * 60 + 777                                   # not a hop multiple
    aud = [synthetic_clip(4, n)]
    host = proc(descriptions=["thunder"], audios=aud)
    frames = int(host.sizes.max())
    assert frames == 1501
    noise = synthetic_noise(1, frames).cuda()
    a = tiny_model.separate(proc(descriptions=["thunder"], audios=aud).to("cuda"), noise=noise)
    b = tiny_model.separate(proc(descriptions=["thunder"], audios=aud).to("cuda"), noise=noise)
    assert a.target[0].shape == (frames * 1920,) and a.residual[0].shape == (frames * 1920,)
    assert torch.isfinite(a.target[0]).all() and torch.isfinite(a.residual[0]).all()
    assert float(a.target[0].abs().max()) <= 1.0
    assert torch.equal(a.target[0], b.target[0]) and torch.equal(a.residual[0], b.residual[0])


def test_separate_30s_clip_vs_oracle(tiny_model, tiny_cfg, tiny_sd):
    """The whole path on a long clip: codec encode, 16 midpoint steps = 32 evaluations at T = 750, codec decode."""
    from oracle import restate
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_noise, synthetic_text_features
    proc = SAMAudioProcessor(1920, 48000)
    aud, desc = [synthetic_clip(7, 48000 * 30)], ["dog barking"]
    host = proc(descriptions=desc, audios=aud)
    noise = synthetic_noise(1, 750)
    out = tiny_model.separate(proc(descriptions=desc, audios=aud).to("cuda"), noise=noise.cuda())
    lat = tiny_model._last_latent.cpu()
    tf, tm = synthetic_text_features(desc)
    tgt, res, ref_lat = restate.separate(tiny_sd, tiny_cfg, host.audios, host.audio_pad_mask, host.sizes, tf, tm,
                                         host.anchor_ids, host.anchor_alignment, noise, return_latent=True)
    cos = float(torch.nn.functional.cosine_similarity(lat.flatten().double(), ref_lat.flatten().double(), dim=0))
    assert out.target[0].shape == (48000 * 30,)
    assert rel_l2(lat, ref_lat) < 5e-2 and cos > 0.998
    assert snr_db(out.target[0].cpu(), tgt[0]) > 30.0 and snr_db(out.residual[0].cpu(), res[0]) > 30.0


def test_candidates_share_their_clips_pad_mask_at_long_T(tiny_model):
    """reranking_candidates = 2 at T = 750 in a ragged batch: the streaming kernel reads the pad mask of clip
    item / candidates.  Candidates with duplicated noise rows equal each other and the single-candidate run."""
    from sam_audio_b200 import SAMAudioProcessor
    from sam_audio_b200.synthetic import synthetic_clip, synthetic_descriptions, synthetic_noise
    proc = SAMAudioProcessor(1920, 48000)
    auds = [synthetic_clip(0, 48000 * 12), synthetic_clip(1, 48000 * 30)]     # the ragged clip comes first
    desc = synthetic_descriptions(2)
    noise = synthetic_noise(2, 750).cuda()
    one = tiny_model.separate(proc(descriptions=desc, audios=auds).to("cuda"), noise=noise)
    two = tiny_model.separate(proc(descriptions=desc, audios=auds).to("cuda"), noise=noise.repeat_interleave(2, 0),
                              reranking_candidates=2)
    for i in range(2):
        assert torch.equal(one.target[i], two.target[i]) and torch.equal(one.residual[i], two.residual[i])


def test_streaming_tc_attention_bounded_large_logits(capi):
    """The bounded softmax sums p = 2^s over the key blocks with no running maximum: logits up to about +-40 in the
    log2 domain.  Item 0's large terms sit in different key blocks for different rows (the sign of the keys' common
    component changes per block); item 1's keys all point one way, so half of its rows see only strongly negative
    logits (every p <= 2^-15) and the other half only strongly positive ones."""
    items, heads, T = 2, 2, 1500
    g = torch.Generator(device="cuda").manual_seed(40)
    u = torch.randint(0, 2, (heads * 128,), device="cuda", generator=g).float() * 2 - 1      # |u|^2 = 128 per head
    key_block = torch.arange(T, device="cuda") // 128
    a0 = torch.where(key_block % 3 == 0, 1.0, -1.0) * (0.6 + 0.4 * torch.rand(T, device="cuda", generator=g))
    a1 = 0.5 + 0.5 * torch.rand(T, device="cuda", generator=g)
    a = torch.stack([a0, a1])                                                                  # [items, T]
    k = (a[..., None] * u + 0.05 * torch.randn(items, T, heads * 128, device="cuda", generator=g)).reshape(items * T, -1)
    b = torch.where(torch.arange(T, device="cuda") % 2 == 0, 38.0, -38.0)
    q = ((b[None, :, None] * u / 128).expand(items, T, heads * 128)
         + 0.01 * torch.randn(items, T, heads * 128, device="cuda", generator=g)).reshape(items * T, -1)
    qs, k = q.bfloat16(), k.bfloat16()                      # q is already in the log2 domain
    v = torch.randn(items * T, heads * 128, device="cuda", generator=g).bfloat16()
    mask = _ragged_mask(items, T)
    ref, s = _reference(qs, k, v, mask, items, heads, T, LN2)
    smax = float(s[torch.isfinite(s)].abs().max()) / LN2
    assert 30.0 < smax < 50.0
    neg_rows = (s[1] / LN2).masked_fill(~torch.isfinite(s[1]), -100.0).amax(-1) < -15.0       # [heads, T]
    assert int(neg_rows.sum()) >= heads * T // 2 - heads
    del s
    o = torch.full((items * T, heads * 128), float("nan"), device="cuda", dtype=torch.bfloat16)
    capi.check(capi.lib().sab_test_attention_stream(items, heads, T, qs.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                    mask.data_ptr(), o.data_ptr(), 0.0, 3, capi.stream_ptr()))
    torch.cuda.synchronize()
    assert torch.isfinite(o.float()).all()
    assert rel_l2(o.float(), ref) < 1e-2
    sel = neg_rows.t().reshape(T, heads, 1).expand(T, heads, 128).reshape(T, heads * 128)     # item 1's negative rows
    assert rel_l2(o.float()[T:][sel], ref[T:][sel]) < 1e-2


def test_streaming_tc_attention_bounded_vs_mma_sync_kernel_and_fully_masked_item(capi):
    """The bounded variant against attention_kernel: the operands differ by the bf16 rounding of the pre-scaled q, so
    the bar is the fp32 one (1e-2), not the 3e-3 of identical inputs.  Item 2 has no valid key at all: the streaming
    kernel writes zeros for it (never 0 * inf)."""
    items, heads, T = 3, 2, 700
    g = torch.Generator(device="cuda").manual_seed(70)
    q, k, v = (torch.randn(items * T, heads * 128, device="cuda", generator=g).bfloat16() for _ in range(3))
    qs = (q.float() * (LOG2E / 128 ** 0.5)).bfloat16()
    mask = _ragged_mask(items, T)
    a = torch.full((items * T, heads * 128), float("nan"), device="cuda", dtype=torch.bfloat16)
    b = torch.full_like(a, float("nan"))
    capi.check(capi.lib().sab_test_attention(items, heads, T, T, q.data_ptr(), k.data_ptr(), v.data_ptr(),
                                             mask.data_ptr(), b.data_ptr(), capi.stream_ptr()))
    capi.check(capi.lib().sab_test_attention_stream(items, heads, T, qs.data_ptr(), k.data_ptr(), v.data_ptr(),
                                                    mask.data_ptr(), a.data_ptr(), 0.0, 0, capi.stream_ptr()))
    torch.cuda.synchronize()
    assert rel_l2(a.float(), b.float()) < 1e-2
    mask[2] = 0
    for shift in (0.0, -1.0):
        a.fill_(float("nan"))
        capi.check(capi.lib().sab_test_attention_stream(items, heads, T, (qs if shift == 0.0 else q).data_ptr(), k.data_ptr(),
                                                        v.data_ptr(), mask.data_ptr(), a.data_ptr(), shift, 3, capi.stream_ptr()))
        torch.cuda.synchronize()
        assert torch.isfinite(a.float()).all() and float(a[2 * T:].float().abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------------------------
# time-tiled codec: a clip that does not fit the workspace budget is cut into tiles with halos
# ---------------------------------------------------------------------------------------------------------------
SMALL_BUDGET = "6e8"      # by the planner's constants: encoder tiles of 267 frames, decoder tiles of 88


def _halo_from_config(codec, decoder):
    """The receptive-field walk of the layer list, restated: 7-tap first / last convs, three residual units per block
    (7 taps, dilations 1 / 3 / 9, then 1 x 1), (transposed) convs of kernel 2 x stride, a 3-tap encoder output conv."""
    res = 3 * (1 + 3 + 9)
    if decoder:
        r = 3
        for s in reversed(codec.decoder_rates):
            r = -(-(r + res) // s) + 1
        return r + 3
    r = 1
    for s in reversed(codec.encoder_rates):
        r = (r + 1) * s + res
    return -(-(r + 3) // codec.hop_length)


def _tile_count(T, Lt, halo):
    n, w0 = 0, 0
    while True:
        start = 0 if w0 == 0 else w0 - halo
        n += 1
        if start + Lt >= T:
            return n
        w0 = start + Lt - halo


def test_codec_halo_and_tile_length_follow_from_the_layer_list(tiny_model, tiny_cfg, monkeypatch):
    eng = tiny_model._ensure_engine()
    for decoder in (False, True):
        halo, tile = eng.codec_tiling(decoder, 750)
        assert halo == _halo_from_config(tiny_cfg.audio_codec, decoder) and tile == 0      # default budget: whole clips
    monkeypatch.setenv("SAB_CODEC_CHUNK_BYTES", SMALL_BUDGET)
    assert eng.codec_tiling(False, 750) == (_halo_from_config(tiny_cfg.audio_codec, False), 267)
    assert eng.codec_tiling(True, 750) == (_halo_from_config(tiny_cfg.audio_codec, True), 88)
    assert eng.codec_tiling(True, 80)[1] == 0                                              # shorter than a tile


@pytest.mark.parametrize("T,enc_tiles,dec_tiles", [(750, 3, 11), (400, 2, 6), (150, 1, 2), (271, 2, 4)])
def test_codec_tiled_equals_untiled_bit_for_bit(tiny_model, tiny_cfg, monkeypatch, T, enc_tiles, dec_tiles):
    """Two clips (the second shorter, zero-padded to the batch length, its length not a hop multiple) encoded and
    decoded under the default budget and under one that forces time tiles: >= 3 tiles, exactly 2, a last tile that
    overlaps its neighbour almost entirely (T = 271 against 267-frame tiles), and a clip too short to tile."""
    from sam_audio_b200.synthetic import synthetic_clip
    eng = tiny_model._ensure_engine()
    n = T * 1920 - 300
    wav = torch.stack([synthetic_clip(1, n), torch.nn.functional.pad(synthetic_clip(2, n - 50000), (0, 50000))]).cuda()
    lat = torch.randn(2, T, 256, generator=torch.Generator().manual_seed(T)).cuda()
    feats = tiny_model._get_audio_features(wav)
    full = torch.empty(2, 2, T * 1920, device="cuda")
    eng.decode(lat, 2, T, full)
    monkeypatch.setenv("SAB_CODEC_CHUNK_BYTES", SMALL_BUDGET)
    for decoder, want in ((False, enc_tiles), (True, dec_tiles)):
        halo, tile = eng.codec_tiling(decoder, T)
        assert (_tile_count(T, tile, halo) if tile else 1) == want
    feats_t = tiny_model._get_audio_features(wav)
    tiled = torch.full_like(full, float("nan"))
    eng.decode(lat, 2, T, tiled)
    torch.cuda.synchronize()
    assert feats.shape == (2, T, 256) and torch.equal(feats, feats_t)
    assert torch.equal(full, tiled)
    assert not torch.equal(tiled[:, 0], tiled[:, 1])           # residual is not a copy of the target


def test_codec_tiled_vs_oracle(tiny_model, tiny_cfg, tiny_sd, monkeypatch):
    from oracle import restate
    from sam_audio_b200.synthetic import synthetic_clip
    T = 300
    monkeypatch.setenv("SAB_CODEC_CHUNK_BYTES", SMALL_BUDGET)
    eng = tiny_model._ensure_engine()
    assert eng.codec_tiling(False, T)[1] > 0 and eng.codec_tiling(True, T)[1] > 0
    wav = torch.stack([synthetic_clip(5, T * 1920 - 700)])
    ref = restate.codec_encode(tiny_sd, tiny_cfg.audio_codec, wav).transpose(1, 2)
    feats = tiny_model._get_audio_features(wav.cuda())
    assert rel_l2(feats[:, :, :128].cpu(), ref) < 2e-2
    lat = torch.randn(1, T, 256, generator=torch.Generator().manual_seed(8))
    ref_w = restate.codec_decode(tiny_sd, tiny_cfg.audio_codec, lat.transpose(1, 2).reshape(2, 128, T)).view(1, 2, -1)
    out = torch.empty(1, 2, T * 1920, device="cuda")
    eng.decode(lat.cuda(), 1, T, out)
    torch.cuda.synchronize()
    assert rel_l2(out.cpu(), ref_w) < 3e-2 and float(out.abs().max()) <= 1.0


def test_codec_workspace_is_bounded_by_the_tile_not_the_clip(tiny_cfg, tiny_sd, monkeypatch):
    """A fresh engine (no other codec plan resident): decoding a 30 s clip in tiles allocates one plan of tile length;
    a 60 s clip afterwards reuses it, so the workspace does not grow at all, while the un-tiled plans of the same clips
    are several times larger and grow with the clip."""
    from sam_audio_b200.model import SAMAudio
    from sam_audio_b200.text_encoder import SyntheticTextEncoder
    m = SAMAudio(tiny_cfg, text_encoder=SyntheticTextEncoder())
    m.load_state_dict(tiny_sd)
    eng = m.eval().cuda()._ensure_engine()

    def decode(T):
        out = torch.empty(1, 2, T * 1920, device="cuda")
        eng.decode(torch.randn(1, T, 256, device="cuda"), 1, T, out)
        torch.cuda.synchronize()
        return eng.workspace_bytes()
    w0 = eng.workspace_bytes()
    monkeypatch.setenv("SAB_CODEC_CHUNK_BYTES", SMALL_BUDGET)
    halo, tile = eng.codec_tiling(True, 750)
    w30 = decode(750)
    w60 = decode(1500)
    monkeypatch.delenv("SAB_CODEC_CHUNK_BYTES")
    u30 = decode(750) - w60
    u60 = decode(1500) - w60 - u30
    one_tile = w30 - w0
    assert w60 - w30 < one_tile and w60 == w30
    assert one_tile < u30 * (tile + 8) / 750 * 1.25           # a plan of `tile` frames, not of 750
    assert u60 > 1.9 * u30                                     # what the un-tiled plan of the longer clip costs
