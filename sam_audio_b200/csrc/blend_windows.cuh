// Cross-fade of overlapping windows: a recording longer than the model's position table is solved as windows of Tw
// frames (SAMAudio.separate, DESIGN.md section 3), and this kernel blends the windowed latents back into one latent per
// sequence:
//   out[s, t, :] = sum_k w_k(t - start_k) * x_k[t - start_k, :] / sum_k w_k(t - start_k)
// over the windows k of sequence s that cover frame t, in ascending window order, with fp32 accumulation.  The weight at
// local position j is min(ramp_in, ramp_out), ramp_in = min(1, (j + 0.5) / O) (1 for the clip's first window) and
// ramp_out = min(1, (Tw - j - 0.5) / O) (1 for its last).  Frames no window covers are written as 0.
//
// HBM-bound: one warp owns BW_FRAMES consecutive frames of one sequence, finds the windows that touch them with one
// ballot per 32 windows, and reads each covering window row once (two float4 per lane per frame).  Every output frame is
// written by exactly one warp and there are no atomics, so the result is reproducible.
#pragma once
#include "common.cuh"

namespace sab {

constexpr int BW_FRAMES = 4;   // frames per warp
constexpr int BW_WARPS = 8;    // warps per CTA
constexpr int BW_FIRST = 1, BW_LAST = 2;

struct BlendParams {
  const float* win;        // [n_win, Tw, 256]
  const int* seq;          // [n_win] destination sequence
  const int* start;        // [n_win] first frame of the window in its sequence
  const uint8_t* flags;    // [n_win] BW_FIRST | BW_LAST
  int n_win, Tw, ramp;
  float* out;              // [Bc, T, 256]
  int T;
};

__global__ void __launch_bounds__(BW_WARPS * 32) blend_windows_kernel(BlendParams p) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int s = blockIdx.y;
  const int t0 = (blockIdx.x * BW_WARPS + warp) * BW_FRAMES;
  if (t0 >= p.T) return;
  const int nf = min(BW_FRAMES, p.T - t0);
  float4 acc[BW_FRAMES][2];
  float wsum[BW_FRAMES];
#pragma unroll
  for (int f = 0; f < BW_FRAMES; ++f) {
    acc[f][0] = acc[f][1] = make_float4(0.f, 0.f, 0.f, 0.f);
    wsum[f] = 0.f;
  }
  const float ramp = (float)p.ramp;
  for (int base = 0; base < p.n_win; base += 32) {
    const int k = base + lane;
    int st = 0;
    bool hit = false;
    if (k < p.n_win) {
      st = __ldg(p.start + k);
      hit = __ldg(p.seq + k) == s && (long long)st < (long long)t0 + nf && (long long)st + p.Tw > t0;
    }
    unsigned m = __ballot_sync(0xffffffffu, hit);
    while (m) {                                     // ascending window order
      const int b = __ffs(m) - 1;
      m &= m - 1;
      const int kw = base + b;
      const int stk = __shfl_sync(0xffffffffu, st, b);
      const int fl = __ldg(p.flags + kw);
      const float* xw = p.win + (long long)kw * p.Tw * 256 + lane * 4;
#pragma unroll
      for (int f = 0; f < BW_FRAMES; ++f) {
        const long long j = (long long)t0 + f - stk;
        if (f >= nf || j < 0 || j >= p.Tw) continue;   // warp-uniform
        const float rin = (fl & BW_FIRST) ? 1.f : fminf(1.f, ((float)j + 0.5f) / ramp);
        const float rout = (fl & BW_LAST) ? 1.f : fminf(1.f, ((float)(p.Tw - j) - 0.5f) / ramp);
        const float w = fminf(rin, rout);
        const float4 a = ldg_stream128(xw + j * 256), c = ldg_stream128(xw + j * 256 + 128);
        acc[f][0].x = fmaf(w, a.x, acc[f][0].x); acc[f][0].y = fmaf(w, a.y, acc[f][0].y);
        acc[f][0].z = fmaf(w, a.z, acc[f][0].z); acc[f][0].w = fmaf(w, a.w, acc[f][0].w);
        acc[f][1].x = fmaf(w, c.x, acc[f][1].x); acc[f][1].y = fmaf(w, c.y, acc[f][1].y);
        acc[f][1].z = fmaf(w, c.z, acc[f][1].z); acc[f][1].w = fmaf(w, c.w, acc[f][1].w);
        wsum[f] += w;
      }
    }
  }
#pragma unroll
  for (int f = 0; f < BW_FRAMES; ++f) {
    if (f >= nf) continue;
    float* o = p.out + ((long long)s * p.T + t0 + f) * 256 + lane * 4;
    const float4 a = acc[f][0], c = acc[f][1];
    const float ws = wsum[f];
    if (ws > 0.f) {
      *reinterpret_cast<float4*>(o) = make_float4(a.x / ws, a.y / ws, a.z / ws, a.w / ws);
      *reinterpret_cast<float4*>(o + 128) = make_float4(c.x / ws, c.y / ws, c.z / ws, c.w / ws);
    } else {                                        // no window covers the frame (pad past the clip's end)
      *reinterpret_cast<float4*>(o) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(o + 128) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

}  // namespace sab
