// Small kernels of the T5 text encoder (reference: sam_audio/model/text_encoder.py:11-37 wraps HF T5EncoderModel;
// arithmetic = transformers' T5Stack: T5LayerNorm (RMS, eps 1e-6), un-scaled dot-product attention with a
// bucketed relative position bias, DenseReluDense).  The linears run on the wgmma GEMM; text is a handful of
// tokens, so these kernels are latency- not throughput-critical.
#pragma once
#include "common.cuh"

namespace sab {

// x[r, :] = emb[ids[r], :]
__global__ void t5_embed_kernel(const long long* __restrict__ ids, const float* __restrict__ emb, int d, long long rows,
                                float* __restrict__ x) {
  const long long n4 = rows * (d / 4);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / (d / 4);
    const int c = (int)(i % (d / 4));
    reinterpret_cast<float4*>(x)[i] = reinterpret_cast<const float4*>(emb + ids[r] * d)[c];
  }
}

// T5LayerNorm: y = x * rsqrt(mean(x^2) + eps) * w ; one warp per row; bf16 and/or fp32 output
__global__ void __launch_bounds__(256)
t5_norm_kernel(const float* __restrict__ x, const float* __restrict__ w, int d, long long rows, float eps,
               __nv_bfloat16* __restrict__ out_bf16, float* __restrict__ out_f32) {
  const long long row = blockIdx.x * 8LL + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* xr = x + row * d;
  float ss = 0.f;
  for (int c = lane; c < d; c += 32) ss = fmaf(xr[c], xr[c], ss);
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss / (float)d + eps);
  for (int c = lane; c < d; c += 32) {
    const float y = xr[c] * rstd * w[c];
    if (out_bf16) out_bf16[row * d + c] = __float2bfloat16(y);
    if (out_f32) out_f32[row * d + c] = y;
  }
}

// Self-attention of one (batch, head): head_dim 64, no 1/sqrt(d) scaling, additive relative position bias
// bias[h][j - i + L - 1], key padding mask.  One warp per query row: lanes own keys in phase 1 (scores),
// dims in phase 2 (P V).  K/V rows are padded to 66 bf16 so that lanes reading different keys hit different banks.
constexpr int T5_HD = 64, T5_LDK = 66, T5_MAX_L = 512;
__global__ void __launch_bounds__(128)
t5_attention_kernel(const __nv_bfloat16* __restrict__ qkv /*[B*L, 3*H*64]*/, const float* __restrict__ bias /*[H, 2L-1]*/,
                    const uint8_t* __restrict__ mask /*[B, L]*/, int L, int H, __nv_bfloat16* __restrict__ out /*[B*L, H*64]*/) {
  extern __shared__ __align__(16) uint8_t t5_smem[];
  __nv_bfloat16* sK = reinterpret_cast<__nv_bfloat16*>(t5_smem);       // [L][66]
  __nv_bfloat16* sV = sK + (size_t)L * T5_LDK;                         // [L][66]
  float* sQ = reinterpret_cast<float*>(sV + (size_t)L * T5_LDK);       // [4 warps][64]
  float* sP = sQ + 4 * T5_HD;                                          // [4 warps][L]
  const int b = blockIdx.y, h = blockIdx.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ld = 3 * H * T5_HD;
  const __nv_bfloat16* base = qkv + (long long)b * L * ld + h * T5_HD;
  for (int i = tid; i < L * (T5_HD / 2); i += 128) {
    const int j = i / (T5_HD / 2), c = (i % (T5_HD / 2)) * 2;
    *reinterpret_cast<uint32_t*>(sK + j * T5_LDK + c) = *reinterpret_cast<const uint32_t*>(base + (long long)j * ld + H * T5_HD + c);
    *reinterpret_cast<uint32_t*>(sV + j * T5_LDK + c) = *reinterpret_cast<const uint32_t*>(base + (long long)j * ld + 2 * H * T5_HD + c);
  }
  __syncthreads();
  const float* brow = bias + (long long)h * (2 * L - 1) + (L - 1);
  const uint8_t* mrow = mask + (long long)b * L;
  float* q = sQ + warp * T5_HD;
  float* pr = sP + warp * L;
  for (int i = warp; i < L; i += 4) {
    const float2 q2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(base + (long long)i * ld + 2 * lane));
    q[2 * lane] = q2.x;
    q[2 * lane + 1] = q2.y;
    __syncwarp();
    float mx = -INFINITY;
    for (int j = lane; j < L; j += 32) {
      float s = 0.f;
      const __nv_bfloat16* kr = sK + j * T5_LDK;
#pragma unroll
      for (int c = 0; c < T5_HD; c += 2) {
        const float2 k2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(kr + c));
        s = fmaf(q[c], k2.x, s);
        s = fmaf(q[c + 1], k2.y, s);
      }
      s = mrow[j] ? s + brow[j - i] : -INFINITY;
      pr[j] = s;
      mx = fmaxf(mx, s);
    }
    mx = warp_max(mx);
    float sum = 0.f;
    for (int j = lane; j < L; j += 32) {
      const float p = __expf(pr[j] - mx);
      pr[j] = p;
      sum += p;
    }
    sum = warp_sum(sum);
    __syncwarp();
    float o0 = 0.f, o1 = 0.f;
    for (int j = 0; j < L; ++j) {
      const float p = pr[j];
      const float2 v2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(sV + j * T5_LDK + 2 * lane));
      o0 = fmaf(p, v2.x, o0);
      o1 = fmaf(p, v2.y, o1);
    }
    const float inv = 1.f / sum;
    *reinterpret_cast<uint32_t*>(out + ((long long)b * L + i) * (H * T5_HD) + h * T5_HD + 2 * lane) = pack_bf16(o0 * inv, o1 * inv);
    __syncwarp();
  }
}

// bias[h][delta] = rel_bias_weight[bucket[delta]][h]  for delta index 0 .. 2L-2
__global__ void t5_bias_table_kernel(const float* __restrict__ w /*[buckets, H]*/, const int* __restrict__ bucket /*[2L-1]*/,
                                     int n_delta, int H, float* __restrict__ bias /*[H, n_delta]*/) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n_delta * H) return;
  const int h = idx / n_delta, dlt = idx % n_delta;
  bias[idx] = w[bucket[dlt] * H + h];
}

}  // namespace sab
