// SIMT kernels at the two 1-channel ends of the DAC-VAE codec, plus layout helpers.
// The multi-channel convolutions run on the wgmma GEMM (gemm_tc.cuh) over channels-last audio.
// (DAC-VAE arithmetic is restated from the Descript-DAC layout; reference call sites codec.py:65-89.)
#pragma once
#include "common.cuh"

namespace sab {

SAB_DEVICE float snake_f(float v, float a) {
  const float s = __sinf(a * v);
  return v + s * s * __frcp_rn(a + 1e-9f);
}

// encoder.block.0: Conv1d(1 -> C0, k=7, pad=3) on mono PCM, output channels-last.
//   x_out[b,t,c] = bias[c] + sum_k w[c,k] * wav[b,t+k-3]        (fp32 residual stream)
//   a_out[b,t,c] = bf16(Snake_alpha(x_out))                      (operand of the first residual unit)
// 16 threads per sample (4 channels each, C0 = 64): 256 B / 128 B coalesced stores per sample.
__global__ void __launch_bounds__(256)
enc_conv0_kernel(const float* __restrict__ wav, long long S, int C0, const float* __restrict__ w /*[C0,7]*/,
                 const float* __restrict__ bias, const float* __restrict__ alpha, float* __restrict__ x_out,
                 __nv_bfloat16* __restrict__ a_out) {
  const int tpc = C0 / 4;  // threads per sample
  const int b = blockIdx.y;
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  const long long t = idx / tpc;
  const int c = (int)(idx % tpc) * 4;
  if (t >= S) return;
  const float* wp = wav + b * S;
  float xin[7];
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const long long tt = t + k - 3;
    xin[k] = (tt >= 0 && tt < S) ? wp[tt] : 0.f;
  }
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float acc = bias[c + j];
#pragma unroll
    for (int k = 0; k < 7; ++k) acc = fmaf(w[(c + j) * 7 + k], xin[k], acc);
    v[j] = acc;
  }
  const long long o = (b * S + t) * C0 + c;
  *reinterpret_cast<float4*>(x_out + o) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<uint2*>(a_out + o) =
      make_uint2(pack_bf16(snake_f(v[0], alpha[c]), snake_f(v[1], alpha[c + 1])),
                 pack_bf16(snake_f(v[2], alpha[c + 2]), snake_f(v[3], alpha[c + 3])));
}

// Same layer with the 4 x 7 weights, bias and Snake constants of the thread's channels held in registers over
// ENC0_ITER samples (requires 256 % (C0/4) == 0): the loads per sample drop from 43 to 7 (the PCM window, L1 hits).
constexpr int ENC0_ITER = 8;
__global__ void __launch_bounds__(256)
enc_conv0_reg_kernel(const float* __restrict__ wav, long long S, int C0, const float* __restrict__ w /*[C0,7]*/,
                     const float* __restrict__ bias, const float* __restrict__ alpha, float* __restrict__ x_out,
                     __nv_bfloat16* __restrict__ a_out) {
  const int tpc = C0 / 4;                      // threads per sample
  const int spb = 256 / tpc;                   // samples per block and iteration
  const int c = (threadIdx.x % tpc) * 4;
  const int sl = threadIdx.x / tpc;
  const long long b = blockIdx.y;
  const long long tb = blockIdx.x * (long long)(spb * ENC0_ITER);
  float wr[4][7], bs[4], al[4], ia[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int k = 0; k < 7; ++k) wr[j][k] = w[(c + j) * 7 + k];
    bs[j] = bias[c + j];
    al[j] = alpha[c + j];
    ia[j] = __frcp_rn(al[j] + 1e-9f);
  }
  const float* wp = wav + b * S;
#pragma unroll 2
  for (int it = 0; it < ENC0_ITER; ++it) {
    const long long t = tb + (long long)it * spb + sl;
    if (t >= S) break;
    float xin[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      const long long tt = t + k - 3;
      xin[k] = (tt >= 0 && tt < S) ? __ldg(wp + tt) : 0.f;
    }
    float v[4], sn[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float acc = bs[j];
#pragma unroll
      for (int k = 0; k < 7; ++k) acc = fmaf(wr[j][k], xin[k], acc);
      v[j] = acc;
      const float s = __sinf(al[j] * acc);
      sn[j] = acc + s * s * ia[j];
    }
    const long long o = (b * S + t) * C0 + c;
    *reinterpret_cast<float4*>(x_out + o) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<uint2*>(a_out + o) = make_uint2(pack_bf16(sn[0], sn[1]), pack_bf16(sn[2], sn[3]));
  }
}

// decoder last layer: Conv1d(C -> 1, k=7, pad=3) + tanh on the Snake-activated channels-last input.
//   wav[i,t] = tanh(bias + sum_{k,c} w[c,k] * a[i,t+k-3,c])
// CTA = 128 samples (+6 halo) staged in shared memory (row padded by 2 bf16 -> conflict-free column reads).
constexpr int DEC_LAST_TB = 128;
__global__ void __launch_bounds__(DEC_LAST_TB)
dec_last_kernel(const __nv_bfloat16* __restrict__ a, long long S, int C, const float* __restrict__ w /*[C,7]*/,
                const float* __restrict__ bias, float* __restrict__ wav) {
  extern __shared__ __align__(16) uint8_t dl_smem[];
  const int ldc = C + 2;
  __nv_bfloat16* sa = reinterpret_cast<__nv_bfloat16*>(dl_smem);           // [(TB+6), ldc]
  float* sw = reinterpret_cast<float*>(sa + (DEC_LAST_TB + 6) * ldc + 2);  // [7, C] (k-major)
  const int item = blockIdx.y;
  const long long t0 = blockIdx.x * (long long)DEC_LAST_TB;
  for (int i = threadIdx.x; i < C * 7; i += DEC_LAST_TB) {
    const int c = i / 7, k = i % 7;
    sw[k * C + c] = w[i];
  }
  const int c2 = C / 2;
  for (int i = threadIdx.x; i < (DEC_LAST_TB + 6) * c2; i += DEC_LAST_TB) {
    const int r = i / c2, cc = (i % c2) * 2;
    const long long t = t0 + r - 3;
    uint32_t v = 0;
    if (t >= 0 && t < S) v = *reinterpret_cast<const uint32_t*>(a + ((long long)item * S + t) * C + cc);
    *reinterpret_cast<uint32_t*>(sa + r * ldc + cc) = v;
  }
  __syncthreads();
  const long long t = t0 + threadIdx.x;
  if (t >= S) return;
  float acc = bias[0];
#pragma unroll
  for (int k = 0; k < 7; ++k) {
    const __nv_bfloat16* row = sa + (threadIdx.x + k) * ldc;
    const float* wk = sw + k * C;
    for (int c = 0; c < C; c += 2) {
      const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(row + c));
      acc = fmaf(f.x, wk[c], acc);
      acc = fmaf(f.y, wk[c + 1], acc);
    }
  }
  wav[(long long)item * S + t] = tanhf(acc);
}

// Same layer, register-blocked (C = 32*NCH <= 128): eight lanes walk one segment of DEC_SEG samples, each holding
// the 7 x C/8 weights of its channels (lane l owns channels 32j + 4l .. +3 of every 32-channel chunk j, so the
// eight 8-byte loads of a chunk form one 64 B line).  Every input row is read once (+6 halo rows per segment),
// feeds seven running sums out[r-3 .. r+3] with 7*C/8 FMAs per lane, and the finished sum out[r-3] is reduced
// over the eight lanes; results leave in groups of eight consecutive samples (one 32 B sector per octet).
constexpr int DEC_SEG = 128;
template <int NCH>
__global__ void __launch_bounds__(256)
dec_last_reg_kernel(const __nv_bfloat16* __restrict__ a, long long S, const float* __restrict__ w /*[C,7]*/,
                    const float* __restrict__ bias, float* __restrict__ wav) {
  constexpr int C = 32 * NCH, CPT = 4 * NCH;
  const int l8 = threadIdx.x & 7;
  const unsigned octet = 0xFFu << (threadIdx.x & 24);
  const long long seg = blockIdx.x * 32LL + (threadIdx.x >> 3);
  const long long t0 = seg * DEC_SEG;
  if (t0 >= S) return;                        // the whole octet leaves together
  const long long item = blockIdx.y;
  const long long t_end = (t0 + DEC_SEG < S) ? t0 + DEC_SEG : S;   // this octet produces samples [t0, t_end)
  float wr[7][CPT];
#pragma unroll
  for (int j = 0; j < NCH; ++j)
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int k = 0; k < 7; ++k) wr[k][4 * j + i] = w[(32 * j + 4 * l8 + i) * 7 + k];
  const float b = bias[0];
  const __nv_bfloat16* base = a + item * S * C + 4 * l8;
  auto load_row = [&](long long t, uint2 (&v)[NCH]) {
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      v[j] = make_uint2(0u, 0u);
      if (t >= 0 && t < S) v[j] = __ldg(reinterpret_cast<const uint2*>(base + t * C + 32 * j));
    }
  };
  float s[7];
#pragma unroll
  for (int j = 0; j < 7; ++j) s[j] = 0.f;
  uint2 cur[NCH], nxt[NCH];
  load_row(t0 - 3, cur);
  float keep = 0.f;
#pragma unroll 1
  for (long long r = t0 - 3; r < t_end + 3; ++r) {
    load_row(r + 1 < t_end + 3 ? r + 1 : -1, nxt);
    float x[CPT];
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      x[4 * j] = __uint_as_float(cur[j].x << 16);
      x[4 * j + 1] = __uint_as_float(cur[j].x & 0xffff0000u);
      x[4 * j + 2] = __uint_as_float(cur[j].y << 16);
      x[4 * j + 3] = __uint_as_float(cur[j].y & 0xffff0000u);
    }
    // row r carries tap k of out[r - k + 3]: slot j = 6 - k of the window s[j] = out[r - 3 + j]
#pragma unroll
    for (int k = 0; k < 7; ++k) {
      float d = 0.f;
#pragma unroll
      for (int c = 0; c < CPT; ++c) d = fmaf(wr[k][c], x[c], d);
      s[6 - k] += d;
    }
    const long long to = r - 3;                // out[to] is complete
    if (to >= t0) {
      float v = s[0];
      v += __shfl_xor_sync(octet, v, 1);
      v += __shfl_xor_sync(octet, v, 2);
      v += __shfl_xor_sync(octet, v, 4);
      const int i = (int)(to - t0) & 7;
      if (i == l8) keep = v;
      if (i == 7 || to == t_end - 1) {
        if (l8 <= i) wav[item * S + (to - i) + l8] = tanhf(keep + b);
      }
    }
#pragma unroll
    for (int j = 0; j < 6; ++j) s[j] = s[j + 1];
    s[6] = 0.f;
#pragma unroll
    for (int j = 0; j < NCH; ++j) cur[j] = nxt[j];
  }
}

// latent [Bc, T, 2*Cz] fp32 -> bf16 [2*Bc, T, Cz]  (model.py:291-295: row 2b = target half, 2b+1 = residual half)
__global__ void latent_split_kernel(const float* __restrict__ lat, int T, int Cz, long long n_total,
                                    __nv_bfloat16* __restrict__ out) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Cz);
    const long long r = i / Cz;
    const int t = (int)(r % T);
    const long long item = r / T;  // 2b + half
    const long long b = item >> 1;
    const int half = (int)(item & 1);
    out[i] = __float2bfloat16(lat[(b * T + t) * (2 * Cz) + half * Cz + c]);
  }
}

// [B, C, T] fp32 -> [B, T, C] bf16 (video features arrive channels-first: model.py:191)
__global__ void transpose_cast_kernel(const float* __restrict__ x, int C, int T, long long n_total,
                                      __nv_bfloat16* __restrict__ y) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long r = i / C;
    const int t = (int)(r % T);
    const long long b = r / T;
    y[i] = __float2bfloat16(x[(b * C + c) * T + t]);
  }
}

}  // namespace sab
