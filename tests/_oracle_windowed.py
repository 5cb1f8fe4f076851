"""TEST INFRASTRUCTURE — separate() of a batch longer than the position table, composed from the restated pieces of
oracle/restate.py: codec encode of the whole clip, the midpoint solve of every window on its sliced inputs, the
cross-fade restated in fp64, and codec decode of the blended latent.  The window list comes from
sam_audio_b200.windows.window_layout (which has its own CPU tests); the blend formula is written out here on its own.
"""
from __future__ import annotations

import torch

from oracle import restate


def blend_fp64(win_latent, windows, candidates: int, B: int, T: int, ramp: int):
    """win_latent [len(windows) * c, Tw, C] (window-major, candidate-minor) -> [B * c, T, C] float64:
    sum_k w_k x_k / sum_k w_k over the windows covering each frame, w(j) = min(ramp_in, ramp_out),
    ramp_in = min(1, (j + 1/2) / ramp) unless the window is its clip's first, ramp_out = min(1, (Tw - j - 1/2) / ramp)
    unless it is the last; frames no window covers are 0."""
    _, Tw, C = win_latent.shape
    num = torch.zeros(B * candidates, T, C, dtype=torch.float64)
    den = torch.zeros(B * candidates, T, 1, dtype=torch.float64)
    j = torch.arange(Tw, dtype=torch.float64)
    for i, w in enumerate(windows):
        r_in = torch.ones(Tw, dtype=torch.float64) if w.first else ((j + 0.5) / ramp).clamp(max=1.0)
        r_out = torch.ones(Tw, dtype=torch.float64) if w.last else ((Tw - j - 0.5) / ramp).clamp(max=1.0)
        wt = torch.minimum(r_in, r_out)[:, None]
        for k in range(candidates):
            s = w.clip * candidates + k
            num[s, w.start:w.start + Tw] += wt * win_latent[i * candidates + k].double()
            den[s, w.start:w.start + Tw] += wt
    return torch.where(den > 0, num / den.clamp(min=1e-300), torch.zeros((), dtype=torch.float64))


def separate_windowed(sd, cfg, audios, pad_mask, sizes, text_features, text_mask, anchor_ids, anchor_alignment, noise,
                      windows, Tw: int, ramp: int, candidates: int = 1, n_steps: int = 16, return_latent=False):
    """audios [B, 1, S] fp32, noise [B * c, T, 256]; no video (zeros, model.py:188-189), rankers None (candidate 0).
    Returns (target list, residual list[, latent])."""
    cc = cfg.audio_codec
    feats = restate.codec_encode(sd, cc, audios).transpose(1, 2)
    feats = torch.cat([feats, feats], 2)
    B, T, _ = feats.shape
    c = candidates
    win_lat = []
    for w in windows:
        sl = slice(w.start, w.start + Tw)

        def rep(x):
            return x.unsqueeze(0).expand(c, *x.shape).contiguous()
        fa = dict(audio_features=rep(feats[w.clip, sl]), text_features=rep(text_features[w.clip]),
                  text_mask=rep(text_mask[w.clip]), masked_video_features=torch.zeros(c, cfg.vision_encoder.dim, Tw),
                  anchor_ids=rep(anchor_ids[w.clip]), anchor_alignment=rep(anchor_alignment[w.clip, sl]),
                  audio_pad_mask=rep(pad_mask[w.clip, sl]))

        def field(t, y):
            return restate.samaudio_forward(sd, cfg, y, time=t.expand(y.shape[0]), **fa)
        y0 = noise[w.clip * c:(w.clip + 1) * c, sl]
        win_lat.append(restate.odeint_midpoint(field, y0, n_steps))
    lat = blend_fp64(torch.cat(win_lat, 0), windows, c, B, T, ramp).float()
    Bc = lat.shape[0]
    wavs = restate.codec_decode(sd, cc, lat.transpose(1, 2).reshape(2 * Bc, cc.codebook_dim, T)).view(Bc, 2, -1)
    n = (sizes * cc.hop_length).int()
    tgt = [wavs[b * c, 0, :int(n[b])] for b in range(B)]
    res = [wavs[b * c, 1, :int(n[b])] for b in range(B)]
    return (tgt, res, lat) if return_latent else (tgt, res)
