// Band-limited resampling by a rational factor (sab_resample, DESIGN.md section 3): streams and SAMAudio.resample()
// bring audio at any rate to the codec's rate and back.  With g = gcd(orig, new), o = orig / g, n = new / g, output
// sample q = m * n + j (phase j < n) is
//   y[q] = sum_{k < K} w[j][k] * x[m * o + lo[j] + k]
// over a polyphase table [n, K] built on the host (resample_table in engine.cu, the design of torchaudio's
// sinc_interp_hann).  Input samples outside [0, L) are zero; a segment whose length is unknown (L < 0) treats only
// negative indices so, and the host checks that every other index it reads lies in its buffer.
//
// One launch runs a list of segments.  A CTA owns RS_BLOCK consecutive outputs of one segment: it stages the input span
// those outputs read into shared memory, applying the channel mean as it loads (channels summed in ascending order,
// then divided by C; the sample itself for C = 1), and each thread then runs the K-term fp32 FMA chain of its outputs in
// ascending k.  An output's bits therefore depend only on the signal and the table, never on how the outputs are split
// into segments or CTAs, which is what lets a stream resample chunk by chunk and get the bits of the whole signal.
// The table is stored k-major ([K, n]), so the consecutive outputs of a warp, whose phases are consecutive, read
// adjacent weights.  Tables of at most RS_SMEM_TABLE floats are staged too; larger ones are read through the read-only
// cache, where they stay resident across the CTAs of an SM.
//
// HBM-bound: 4 * C bytes per input sample read (plus the overlap of K samples between neighbouring CTAs), 4 bytes per
// output written.
#pragma once
#include "common.cuh"

namespace sab {

constexpr int RS_THREADS = 256;
constexpr int RS_PER_THREAD = 4;
constexpr int RS_BLOCK = RS_THREADS * RS_PER_THREAD;   // outputs per CTA
constexpr int RS_SMEM_TABLE = 2048;                    // floats: tables up to this size are staged in shared memory
constexpr int RS_MAX_SMEM = 160 * 1024;                // dynamic shared memory the kernel may be launched with

struct ResampleSeg {        // device form of one sab_resample_seg
  const float* in;          // [C, in_count] at channel stride `stride`: signal samples [in_first, in_first + in_count)
  long long stride, in_first, in_count;
  long long length;         // signal length, < 0: unknown
  float* out;               // outputs [out_first, out_first + out_count), contiguous
  long long out_first, out_count;
  const float* w;           // [K, n]: the table k-major, so the phases of a warp's outputs read adjacent floats
  const int* lo;            // [n]
  int o, n, K, C;
  int cta0;                 // first CTA of the segment in the launch
  int smem_table;           // the table is staged in shared memory
};

template <bool kSmemTable>
__device__ __forceinline__ void resample_outputs(const ResampleSeg& s, const float* tab, const float* xs, long long q0,
                                                 int nq, long long i0) {
  const int n = s.n, o = s.o, K = s.K;
  const long long q = q0 + threadIdx.x;
  long long m = q / n;
  int j = (int)(q - m * n);
  const int dm = RS_THREADS / n, dj = RS_THREADS % n;
#pragma unroll
  for (int r = 0; r < RS_PER_THREAD; ++r) {
    const int local = threadIdx.x + r * RS_THREADS;
    if (local < nq) {
      const float* x = xs + (m * o + __ldg(s.lo + j) - i0);
      float acc = 0.f;
      if (kSmemTable) {
        const float* w = tab + j;
#pragma unroll 4
        for (int k = 0; k < K; ++k) acc = fmaf(w[k * n], x[k], acc);
      } else {
        const float* w = s.w + j;
#pragma unroll 4
        for (int k = 0; k < K; ++k) acc = fmaf(__ldg(w + (long long)k * n), x[k], acc);
      }
      s.out[q0 - s.out_first + local] = acc;
    }
    m += dm;
    j += dj;
    if (j >= n) {
      j -= n;
      ++m;
    }
  }
}

// grid: one CTA per RS_BLOCK outputs of every segment (segments in order, segs[i].cta0 ascending);
// dynamic shared memory: tab_floats + the largest input span of any CTA, in floats.
__global__ void __launch_bounds__(RS_THREADS) resample_kernel(const ResampleSeg* __restrict__ segs, int n_segs,
                                                              int tab_floats) {
  extern __shared__ float rs_smem[];
  int a = 0, b = n_segs - 1;                       // the last segment whose first CTA is <= this one
  while (a < b) {
    const int mid = (a + b + 1) >> 1;
    if (segs[mid].cta0 <= (int)blockIdx.x) a = mid;
    else b = mid - 1;
  }
  const ResampleSeg s = segs[a];
  const long long q0 = s.out_first + (long long)(blockIdx.x - s.cta0) * RS_BLOCK;
  const int nq = (int)min((long long)RS_BLOCK, s.out_first + s.out_count - q0);
  const int n = s.n, o = s.o;
  const long long ql = q0 + nq - 1;
  const long long m0 = q0 / n, m1 = ql / n;
  const long long i0 = m0 * o + __ldg(s.lo + (int)(q0 - m0 * n));         // first tap of the first output
  const long long i1 = m1 * o + __ldg(s.lo + (int)(ql - m1 * n)) + s.K;   // one past the last tap of the last output
  float* xs = rs_smem + tab_floats;
  if (s.smem_table)
    for (int t = threadIdx.x; t < n * s.K; t += RS_THREADS) rs_smem[t] = __ldg(s.w + t);
  const long long end = s.length < 0 ? i1 : min(i1, s.length);
  for (long long i = i0 + threadIdx.x; i < i1; i += RS_THREADS) {
    float v = 0.f;
    const long long r = i - s.in_first;
    if (i >= 0 && i < end && r >= 0 && r < s.in_count) {   // the host checked that [0, end) lies in the buffer
      const float* p = s.in + r;
      v = __ldg(p);
      for (int c = 1; c < s.C; ++c) v = v + __ldg(p + c * s.stride);
      if (s.C > 1) v = v / (float)s.C;
    }
    xs[i - i0] = v;
  }
  __syncthreads();
  if (s.smem_table) resample_outputs<true>(s, rs_smem, xs, q0, nq, i0);
  else resample_outputs<false>(s, rs_smem, xs, q0, nq, i0);
}

}  // namespace sab
