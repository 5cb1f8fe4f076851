// Multichannel stems from one mono separation (sab_spread_channels, DESIGN.md section 3).  This goes beyond the
// reference, whose model and examples are mono: the mono target T and residual R of a separation define one
// time-frequency Wiener mask, and that mask is applied to every channel of the mixture, so the stems keep the input's
// spatial image and each channel's target and residual sum to that channel.
//
// At the codec's rate, with N = 2048, hop a = 512 and the periodic Hann window w[n] = 0.5 - 0.5 cos(2 pi n / N):
//   frame j >= 0 covers samples [j a - 3 a, j a + a) (samples outside a signal's known range are zero), so sample
//   s >= 0 lies in exactly the frames floor(s / a) .. floor(s / a) + 3;
//   X_c,j = rfft(w . x_c[frame j]), T_j and R_j likewise;
//   M_j[k] = (|T_j[k]|^2 + d) / (|T_j[k]|^2 + |R_j[k]|^2 + 2 d), d = 1e-10;
//   target_c[s] = (2/3) sum_j w[s - start_j] irfft(M_j X_c,j)[s - start_j] over the four covering frames, ascending j
//   (sum w^2 = 3/2 at hop N/4), and residual_c[s] = x_c[s] - target_c[s], one fp32 subtraction.
//
// One launch runs a list of segments.  A CTA owns SP_HOPS output hops of one segment: it computes every frame that
// covers them, in ascending j, and overlap-adds into shared memory, then writes each of its outputs once.  A sample's
// bits depend only on its four frames, never on how the outputs are cut into segments or CTAs, which is what lets a
// stream spread chunk by chunk and get the bits of the whole recording.
//
// FFTs: radix-2 in shared memory, SP_THREADS threads, twiddles from a table computed once in float64 and rounded to
// fp32 (spread_table_dev in engine.cu).  Two real signals share one complex FFT: T + i R for the mask (separated through
// Z[k] and conj Z[N - k]), and channels pairwise, x_c + i x_c+1.  A channel pair needs no separation: M_j is real and
// M_j[k] = M_j[N - k], so M_j FFT(x_c + i x_c+1) = FFT(y_c + i y_c+1) and one inverse FFT gives both channels' frames.
// The forward FFT is decimation in frequency (natural order in, bit-reversed out) and the inverse decimation in time
// (bit-reversed in, natural out), so no permutation pass is needed; the mask is stored in the bit-reversed order too.
//
// Traffic: T, R and the C channels are read once, plus the (SP_HOPS + 3) / SP_HOPS frame overlap of neighbouring
// CTAs, and the 2 C outputs are written once: 4 (2 + 3 C) bytes per output sample.
#pragma once
#include "common.cuh"

namespace sab {

constexpr int SP_N = 2048;
constexpr int SP_LOG_N = 11;
constexpr int SP_HOP = 512;
constexpr int SP_THREADS = 512;
constexpr int SP_HOPS = 8;                      // output hops per CTA
constexpr int SP_SPAN = SP_HOPS * SP_HOP;       // outputs per CTA and channel
constexpr float SP_DELTA = 1e-10f;
// Z [N] float2, twiddles [N / 2] float2, mask [N] float, then the overlap-add accumulator [C, SP_SPAN] float
constexpr int SP_SMEM_FIXED = SP_N * 8 + SP_N / 2 * 8 + SP_N * 4;
constexpr int SP_MAX_SMEM = SP_SMEM_FIXED + 8 * SP_SPAN * 4;

struct SpreadSeg {          // device form of one sab_spread_seg
  const float* t;           // mono target and residual: samples [tr_first, tr_first + tr_count)
  const float* r;
  long long tr_first, tr_count, tr_length;   // length < 0: unknown
  const float* x;           // [C, x_count] at channel stride x_stride: samples [x_first, x_first + x_count)
  long long x_stride, x_first, x_count, x_length;
  float* ot;                // [C, o_count] at channel stride o_stride: outputs [o_first, o_first + o_count)
  float* orr;
  long long o_stride, o_first, o_count;
  int C;
  int cta0;                 // first CTA of the segment in the launch
};

// Sample i of a window [first, first + count) of a signal of `length` samples (< 0: unknown): zero outside [0, length);
// the host checked that every other index a CTA reads lies in the window.
SAB_DEVICE float sp_sample(const float* p, long long first, long long count, long long length, long long i) {
  if (i < 0 || (length >= 0 && i >= length)) return 0.f;
  const long long r = i - first;
  return (r >= 0 && r < count) ? __ldg(p + r) : 0.f;
}

SAB_DEVICE float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// Forward DFT (exponent -2 pi i k n / N), natural order in, bit-reversed order out.  Ends with a barrier.
SAB_DEVICE void sp_fft_dif(float2* Z, const float2* tw) {
  for (int h = SP_N / 2, step = 1; h >= 1; h >>= 1, step <<= 1) {
    for (int b = threadIdx.x; b < SP_N / 2; b += SP_THREADS) {
      const int off = b & (h - 1), i = ((b - off) << 1) + off;
      const float2 u = Z[i], v = Z[i + h];
      Z[i] = make_float2(u.x + v.x, u.y + v.y);
      Z[i + h] = cmul(make_float2(u.x - v.x, u.y - v.y), tw[off * step]);
    }
    __syncthreads();
  }
}

// Inverse DFT without the 1 / N (exponent +2 pi i k n / N), bit-reversed order in, natural order out; the input is
// first multiplied by the real mask M (in the same bit-reversed order).  Ends with a barrier.
SAB_DEVICE void sp_ifft_dit(float2* Z, const float2* tw, const float* M) {
  for (int h = 1, step = SP_N / 2; h < SP_N; h <<= 1, step >>= 1) {
    for (int b = threadIdx.x; b < SP_N / 2; b += SP_THREADS) {
      const int off = b & (h - 1), i = ((b - off) << 1) + off;
      float2 u = Z[i], v = Z[i + h];
      if (h == 1) {
        u = make_float2(u.x * M[i], u.y * M[i]);
        v = make_float2(v.x * M[i + 1], v.y * M[i + 1]);
      }
      const float2 w = tw[off * step];
      const float2 t = cmul(v, make_float2(w.x, -w.y));
      Z[i] = make_float2(u.x + t.x, u.y + t.y);
      Z[i + h] = make_float2(u.x - t.x, u.y - t.y);
    }
    __syncthreads();
  }
}

SAB_DEVICE int sp_brev(int p) { return (int)(__brev((unsigned)p) >> (32 - SP_LOG_N)); }

// grid: one CTA per SP_HOPS output hops of every segment (segments in order, segs[i].cta0 ascending);
// table: twiddles [N / 2] float2 then the window [N] float; dynamic shared memory SP_SMEM_FIXED + 4 C_max SP_SPAN.
__global__ void __launch_bounds__(SP_THREADS, 2) spread_channels_kernel(const SpreadSeg* __restrict__ segs, int n_segs,
                                                                     const float2* __restrict__ table) {
  extern __shared__ float2 sp_smem[];
  float2* Z = sp_smem;
  float2* tw = Z + SP_N;
  float* M = reinterpret_cast<float*>(tw + SP_N / 2);
  float* acc = M + SP_N;
  const float* win = reinterpret_cast<const float*>(table + SP_N / 2);

  int a = 0, b = n_segs - 1;                       // the last segment whose first CTA is <= this one
  while (a < b) {
    const int mid = (a + b + 1) >> 1;
    if (segs[mid].cta0 <= (int)blockIdx.x) a = mid;
    else b = mid - 1;
  }
  const SpreadSeg s = segs[a];
  const long long h0 = s.o_first / SP_HOP + (long long)(blockIdx.x - s.cta0) * SP_HOPS;
  const long long s0 = max(s.o_first, h0 * SP_HOP);
  const long long s1 = min(s.o_first + s.o_count, (h0 + SP_HOPS) * SP_HOP);
  const int span = (int)(s1 - s0);
  const long long j0 = s0 / SP_HOP, j1 = (s1 - 1) / SP_HOP + 3;

  for (int t = threadIdx.x; t < SP_N / 2; t += SP_THREADS) tw[t] = __ldg(table + t);
  for (int t = threadIdx.x; t < s.C * SP_SPAN; t += SP_THREADS) acc[t] = 0.f;
  __syncthreads();

  for (long long j = j0; j <= j1; ++j) {
    const long long start = j * SP_HOP - 3 * SP_HOP;
    // the mask of frame j from T + i R
    for (int n = threadIdx.x; n < SP_N; n += SP_THREADS) {
      const float w = __ldg(win + n);
      Z[n] = make_float2(w * sp_sample(s.t, s.tr_first, s.tr_count, s.tr_length, start + n),
                         w * sp_sample(s.r, s.tr_first, s.tr_count, s.tr_length, start + n));
    }
    __syncthreads();
    sp_fft_dif(Z, tw);
    for (int p = threadIdx.x; p < SP_N; p += SP_THREADS) {
      int k = sp_brev(p);
      k = k <= SP_N / 2 ? k : SP_N - k;
      const float2 za = Z[sp_brev(k)], zb = Z[sp_brev((SP_N - k) & (SP_N - 1))];
      // T[k] = (Z[k] + conj Z[N - k]) / 2, R[k] = (Z[k] - conj Z[N - k]) / 2i
      const float tr = 0.5f * (za.x + zb.x), ti = 0.5f * (za.y - zb.y);
      const float rr = 0.5f * (za.y + zb.y), ri = 0.5f * (za.x - zb.x);
      const float t2 = tr * tr + ti * ti, r2 = rr * rr + ri * ri;
      M[p] = (t2 + SP_DELTA) / (t2 + r2 + 2.f * SP_DELTA);
    }
    __syncthreads();
    // every channel pair through the mask, overlap-added in ascending j
    for (int c = 0; c < s.C; c += 2) {
      const bool two = c + 1 < s.C;
      const float* x0 = s.x + (long long)c * s.x_stride;
      for (int n = threadIdx.x; n < SP_N; n += SP_THREADS) {
        const float w = __ldg(win + n);
        const long long i = start + n;
        Z[n] = make_float2(w * sp_sample(x0, s.x_first, s.x_count, s.x_length, i),
                           two ? w * sp_sample(x0 + s.x_stride, s.x_first, s.x_count, s.x_length, i) : 0.f);
      }
      __syncthreads();
      sp_fft_dif(Z, tw);
      sp_ifft_dit(Z, tw, M);
      const long long n0 = max(0LL, s0 - start), n1 = min((long long)SP_N, s1 - start);
      for (long long n = n0 + threadIdx.x; n < n1; n += SP_THREADS) {
        const float w = __ldg(win + n);
        const int l = (int)(start + n - s0);
        const float2 y = Z[n];
        acc[c * SP_SPAN + l] = fmaf(w, y.x * (1.f / SP_N), acc[c * SP_SPAN + l]);
        if (two) acc[(c + 1) * SP_SPAN + l] = fmaf(w, y.y * (1.f / SP_N), acc[(c + 1) * SP_SPAN + l]);
      }
      __syncthreads();
    }
  }

  for (int l = threadIdx.x; l < span; l += SP_THREADS) {
    const long long i = s0 + l;
    for (int c = 0; c < s.C; ++c) {
      const float t = acc[c * SP_SPAN + l] * (2.f / 3.f);
      const float xv = sp_sample(s.x + (long long)c * s.x_stride, s.x_first, s.x_count, s.x_length, i);
      s.ot[c * s.o_stride + (i - s.o_first)] = t;
      s.orr[c * s.o_stride + (i - s.o_first)] = xv - t;
    }
  }
}

}  // namespace sab
