// HBM-bound fused elementwise / reduction kernels of the DiT path (float4 loads, warp-shuffle reductions).
// Each kernel cites the reference lines whose arithmetic it fuses.
#pragma once
#include "common.cuh"

namespace sab {

// ---------------------------------------------------------------------------------------------
// RMSNorm + adaLN modulate  (transformer.py:42-47 RMSNorm fp32, :21-22 modulate, :375/:389/:513-515)
//   out[m, :] = bf16( x[m,:] * rsqrt(mean(x^2)+eps) * w * (1 + scale[b,:]) + shift[b,:] ),  b = m / rows_per_item
// one warp per row.
// ---------------------------------------------------------------------------------------------
template <int kVecPerLane>  // d = kVecPerLane * 128
__global__ void __launch_bounds__(256, (kVecPerLane > 24) ? 1 : 2)
rmsnorm_mod_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ shift,
                   const float* __restrict__ scale, long long mod_ld, int rows_per_item,
                   __nv_bfloat16* __restrict__ out, int M, float eps, int reverse) {
  // Single pass: the row lives in registers (kVecPerLane float4 per lane, 88 floats at d = 2816), so x is read from
  // HBM exactly once (6 B per element: 4 read + 2 written).  All of a lane's loads are issued back to back
  // (streaming, no L1 allocation) before the reduction; 2 CTAs x 8 warps per SM keep >100 KB of loads in flight,
  // several times the bandwidth-latency product.  The two-pass version re-read every row (10 B per element).
  constexpr int d = kVecPerLane * 128;
  int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  if (reverse) row = M - 1 - row;      // last rows first: the producer wrote them last, they are still in L2
  const float* xr = x + (long long)row * d + lane * 4;
  float4 v[kVecPerLane];
#pragma unroll
  for (int i = 0; i < kVecPerLane; ++i) v[i] = ldg_stream128(xr + i * 128);
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < kVecPerLane; ++i) ss += v[i].x * v[i].x + v[i].y * v[i].y + v[i].z * v[i].z + v[i].w * v[i].w;
  ss = warp_sum(ss);
  const float rstd = rsqrtf(ss / (float)d + eps);
  const long long b = row / rows_per_item;
  const float4* wr = reinterpret_cast<const float4*>(w);
  const float4* sh = reinterpret_cast<const float4*>(shift + b * mod_ld);
  const float4* sc = reinterpret_cast<const float4*>(scale + b * mod_ld);
  uint2* orow = reinterpret_cast<uint2*>(out + (long long)row * d);
#pragma unroll
  for (int i = 0; i < kVecPerLane; ++i) {
    const int c = lane + i * 32;
    const float4 ww = __ldg(wr + c), s1 = __ldg(sc + c), s0 = __ldg(sh + c);
    const float a = v[i].x * rstd * ww.x * (1.f + s1.x) + s0.x;
    const float bb = v[i].y * rstd * ww.y * (1.f + s1.y) + s0.y;
    const float cc = v[i].z * rstd * ww.z * (1.f + s1.z) + s0.z;
    const float dd = v[i].w * rstd * ww.w * (1.f + s1.w) + s0.w;
    orow[c] = make_uint2(pack_bf16(a, bb), pack_bf16(cc, dd));
  }
}

// ---------------------------------------------------------------------------------------------
// adaLN tables for one NFE  (transformer.py:363-371, :507-509):
//   mod[l][b][r][:] = scale_shift_table_l[r][:] + t0[b][r*d : (r+1)*d],  r = 0..5
//   fin[b][r][:]    = final_table[r][:] + t[b][:],                        r = 0..1
// ---------------------------------------------------------------------------------------------
__global__ void build_mod_kernel(const float* __restrict__ tables /*[L,6,d]*/, const float* __restrict__ t0 /*[B,6d]*/,
                                 float* __restrict__ mod /*[L,B,6,d]*/, int L, int B, int d,
                                 const float* __restrict__ ftable /*[2,d]*/, const float* __restrict__ t /*[B,d]*/,
                                 float* __restrict__ fin /*[B,2,d]*/) {
  const long long n_mod = (long long)L * B * 6 * d / 4;
  const long long n_fin = (long long)B * 2 * d / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_mod + n_fin;
       i += (long long)gridDim.x * blockDim.x) {
    if (i < n_mod) {
      const long long e = i * 4;
      const int c = (int)(e % (6 * d));
      const int b = (int)((e / (6 * d)) % B);
      const int l = (int)(e / ((long long)6 * d * B));
      const float4 a = *reinterpret_cast<const float4*>(tables + (long long)l * 6 * d + c);
      const float4 bb = *reinterpret_cast<const float4*>(t0 + (long long)b * 6 * d + c);
      *reinterpret_cast<float4*>(mod + e) = make_float4(a.x + bb.x, a.y + bb.y, a.z + bb.z, a.w + bb.w);
    } else {
      const long long e = (i - n_mod) * 4;
      const int c = (int)(e % d);
      const int r = (int)((e / d) % 2);
      const int b = (int)(e / (2 * d));
      const float4 a = *reinterpret_cast<const float4*>(ftable + r * d + c);
      const float4 bb = *reinterpret_cast<const float4*>(t + (long long)b * d + c);
      *reinterpret_cast<float4*>(fin + e) = make_float4(a.x + bb.x, a.y + bb.y, a.z + bb.z, a.w + bb.w);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Fused RMSNorm + modulate tables for one NFE (see gemm_tc.cuh): for norm k = 2l (attention_norm of layer l, adaLN rows
// 0/1 = shift_msa/scale_msa) or 2l+1 (ffn_norm, rows 3/4):
//   cs[k][b][:]    = w_norm_k * (1 + scale)          (column scale the producer applies to h)
//   shift[k][b][:] = bf16(shift)                     (A operand of the per-item bias GEMM shift @ W^T)
// ---------------------------------------------------------------------------------------------
__global__ void norm_tables_kernel(const float* __restrict__ mod /*[L,B,6,d]*/, const float* __restrict__ norm_w /*[2L,d]*/,
                                   int L, int B, int d, float* __restrict__ cs /*[2L,B,d]*/,
                                   __nv_bfloat16* __restrict__ shift /*[2L,B,d]*/) {
  const long long n4 = (long long)2 * L * B * d / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const long long e = i * 4;
    const int c = (int)(e % d);
    const int b = (int)((e / d) % B);
    const int k = (int)(e / ((long long)d * B));
    const int l = k >> 1, r0 = (k & 1) * 3;
    const float* m = mod + (((long long)l * B + b) * 6 + r0) * d + c;
    const float4 sh = *reinterpret_cast<const float4*>(m);
    const float4 sc = *reinterpret_cast<const float4*>(m + d);
    const float4 w = *reinterpret_cast<const float4*>(norm_w + (long long)k * d + c);
    *reinterpret_cast<float4*>(cs + e) = make_float4(w.x * (1.f + sc.x), w.y * (1.f + sc.y), w.z * (1.f + sc.z), w.w * (1.f + sc.w));
    *reinterpret_cast<uint2*>(shift + e) = make_uint2(pack_bf16(sh.x, sh.y), pack_bf16(sh.z, sh.w));
  }
}

// ---------------------------------------------------------------------------------------------
// Timestep features (transformer.py:236-253: cat(cos,sin) of t*exp(-ln(1e4) i/128), raw t)  -> bf16 [B,256]
// and the memory input (model.py:30-42,170-172: memory_proj(text) + cat(cos,sin)(t*exp(-ln(1e4) i/(d/2)))) -> bf16 [B*L,d]
// ---------------------------------------------------------------------------------------------
__global__ void tfreq_kernel(const float* __restrict__ time /*[R]*/, int R, __nv_bfloat16* __restrict__ tfreq /*[R,256]*/) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * 256) return;
  const int b = i / 256, c = i % 256;
  const int k = c & 127;
  const float f = expf(-logf(10000.f) * (float)k / 128.f);
  const float a = time[b] * f;
  tfreq[i] = __float2bfloat16(c < 128 ? cosf(a) : sinf(a));
}
// text memory input: memory_proj(text) + cat(cos, sin)(t * exp(-ln(1e4) i/(d/2))) per CLIP; its time is that of the
// clip's first candidate (all equal inside a solve)
__global__ void mem_time_kernel(const float* __restrict__ time /*[B*cand]*/, int B /*sequences*/, int cand, int d, int L,
                                const float* __restrict__ mem_base /*[B/cand*L,d]*/,
                                __nv_bfloat16* __restrict__ mem_in /*[B/cand*L,d]*/) {
  const long long n2 = (long long)(B / cand) * L * d;
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n2; e += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(e % d);
    const int b = (int)(e / ((long long)L * d));
    const int half = d / 2;
    const int k = c < half ? c : c - half;
    const float f = expf(-logf(10000.f) * (float)k / (float)half);
    const float a = time[(long long)b * cand] * f;
    mem_in[e] = __float2bfloat16(mem_base[e] + (c < half ? cosf(a) : sinf(a)));
  }
}

// Runge-Kutta stage combination: out = y + a1 k1 + a2 k2 + a3 k3 + a4 k4 (fp32) and its bf16 copy, the operand of the
// next evaluation's input projection (out may alias y)
__global__ void ode_combine_kernel(const float* y, const float* __restrict__ k1, float a1, const float* __restrict__ k2,
                                   float a2, const float* __restrict__ k3, float a3, const float* __restrict__ k4, float a4,
                                   float* out, __nv_bfloat16* __restrict__ out_bf, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = y[i] + a1 * k1[i];
    if (a2 != 0.f) v += a2 * k2[i];
    if (a3 != 0.f) v += a3 * k3[i];
    if (a4 != 0.f) v += a4 * k4[i];
    out[i] = v;
    out_bf[i] = __float2bfloat16(v);
  }
}

// silu + cast (transformer.py:492 t_block_non_linearity) fp32 -> bf16
__global__ void silu_cast_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16(silu_f(x[i]));
}
__global__ void cast_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = __float2bfloat16(x[i]);
}

// ---------------------------------------------------------------------------------------------
// GroupNorm(1 group) over the whole (T, C) slab of an item, then SiLU  (patcher.py:83-98, num_groups=1)
// pass 1: per-item partial sums (double) ; pass 2: normalise + affine + SiLU -> bf16
// The sums are taken about the item's first element K: var = E[(x-K)^2] - E[x-K]^2 keeps the cancellation of
// E[x^2] - mean^2 away when the item's mean is large next to its spread (mean/std = 300 lost every significant digit
// of the variance in the fp32 per-thread partials; about K the loss scales with ((mean-K)/std)^2 instead).
// ---------------------------------------------------------------------------------------------
constexpr int GN_CHUNKS = 32;
__global__ void __launch_bounds__(256)
gn_stats_kernel(const float* __restrict__ x, long long n_per_item, double* __restrict__ partial /*[items,GN_CHUNKS,2]*/) {
  const int item = blockIdx.y, chunk = blockIdx.x;
  const long long n4 = n_per_item / 4;
  const long long per = (n4 + GN_CHUNKS - 1) / GN_CHUNKS;
  const long long lo = chunk * per, hi = (lo + per < n4) ? lo + per : n4;
  const float4* xp = reinterpret_cast<const float4*>(x + item * n_per_item);
  const float K = x[item * n_per_item];
  float s = 0.f, q = 0.f;
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    float4 v = xp[i];
    v.x -= K; v.y -= K; v.z -= K; v.w -= K;
    s += v.x + v.y + v.z + v.w;
    q += v.x * v.x + v.y * v.y + v.z * v.z + v.w * v.w;
  }
  __shared__ double sh[2][8];
  double ds = warp_sum(s), dq = warp_sum(q);
  // (per-thread fp32 partials over <= a few thousand elements, then double across warps/chunks)
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = ds; sh[1][threadIdx.x >> 5] = dq; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, b = 0;
    for (int i = 0; i < 8; ++i) { a += sh[0][i]; b += sh[1][i]; }
    partial[((long long)item * GN_CHUNKS + chunk) * 2] = a;
    partial[((long long)item * GN_CHUNKS + chunk) * 2 + 1] = b;
  }
}

__global__ void __launch_bounds__(256)
gn_silu_kernel(const float* __restrict__ x, const double* __restrict__ partial, const float* __restrict__ gamma,
               const float* __restrict__ beta, int C, long long n_per_item, float eps,
               __nv_bfloat16* __restrict__ y) {
  const int item = blockIdx.y;
  __shared__ float s_mean, s_rstd;
  if (threadIdx.x == 0) {
    double a = 0, b = 0;
    for (int i = 0; i < GN_CHUNKS; ++i) {
      a += partial[((long long)item * GN_CHUNKS + i) * 2];
      b += partial[((long long)item * GN_CHUNKS + i) * 2 + 1];
    }
    const double dm = a / (double)n_per_item;          // mean - K
    const double var = b / (double)n_per_item - dm * dm;
    s_mean = (float)((double)x[item * n_per_item] + dm);
    s_rstd = (float)(1.0 / sqrt((var > 0 ? var : 0) + (double)eps));
  }
  __syncthreads();
  const float mean = s_mean, rstd = s_rstd;
  const float4* xp = reinterpret_cast<const float4*>(x + item * n_per_item);
  uint2* yp = reinterpret_cast<uint2*>(y + item * n_per_item);
  const long long n4 = n_per_item / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = xp[i];
    const int c = (int)((i * 4) % C);
    const float4 g = *reinterpret_cast<const float4*>(gamma + c);
    const float4 bb = *reinterpret_cast<const float4*>(beta + c);
    const float a0 = silu_f((v.x - mean) * rstd * g.x + bb.x);
    const float a1 = silu_f((v.y - mean) * rstd * g.y + bb.y);
    const float a2 = silu_f((v.z - mean) * rstd * g.z + bb.z);
    const float a3 = silu_f((v.w - mean) * rstd * g.w + bb.w);
    yp[i] = make_uint2(pack_bf16(a0, a1), pack_bf16(a2, a3));
  }
}

// ---------------------------------------------------------------------------------------------
// Conditioning finish, once per separate() call (time-independent part of align_inputs):
//   cond[m,:] += tanh(g_v) * LayerNorm(vproj[m,:]) (or the constant vector for absent video)     align.py:41-50
//             +  tanh(g_a) * E[ ids[b, align[b,t]] , :]        E = embed @ proj^T (4 x d)          model.py:63-65
// one warp per row.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
cond_finish_kernel(float* cond /*[M,d] per sequence*/, const float* cond_clip /*[M/cand,d]; == cond when cand == 1*/,
                   int M, int d, int T, int cand,
                   const float* __restrict__ vproj /*[M/cand,d] or null*/, const float* __restrict__ ln_w,
                   const float* __restrict__ ln_b, const float* __restrict__ vconst /*[d] (used when vproj null)*/,
                   const float* __restrict__ gate_v, const float* __restrict__ anchor_table /*[n_anchor+1, d]*/,
                   const long long* __restrict__ anchor_ids, int n_ids, const long long* __restrict__ anchor_align,
                   const float* __restrict__ gate_a, int video_term, int anchor_term) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= M) return;
  const int b = (row / T) / cand, t = row % T;       // clip of this sequence row
  const long long crow = (long long)b * T + t;
  // forward(masked_video_features=None) / forward(anchor_ids=None) leave the input unchanged (align.py:41-42,
  // model.py:57-58); separate() always supplies both (zeros video = the constant term, <null> anchors)
  const float gv = video_term ? tanhf(gate_v[0]) : 0.f, ga = anchor_term ? tanhf(gate_a[0]) : 0.f;
  const float* er = anchor_table;
  if (anchor_term) {
    const long long slot = anchor_align[crow];
    er = anchor_table + anchor_ids[(long long)b * n_ids + slot] * d;
  }
  float* cr = cond + (long long)row * d;
  const float* ci = cond_clip + crow * d;
  float mean = 0.f, rstd = 0.f;
  const float* vr = nullptr;
  if (vproj && video_term) {
    vr = vproj + crow * d;
    float s = 0.f;
    for (int c = lane; c < d; c += 32) s += vr[c];
    mean = warp_sum(s) / (float)d;
    float q = 0.f;
    for (int c = lane; c < d; c += 32) { const float u = vr[c] - mean; q += u * u; }
    rstd = rsqrtf(warp_sum(q) / (float)d + 1e-5f);
  }
  for (int c = lane; c < d; c += 32) {
    const float vterm = vr ? ((vr[c] - mean) * rstd * ln_w[c] + ln_b[c]) : vconst[c];
    cr[c] = ci[c] + gv * vterm + ga * er[c];
  }
}

// LayerNorm of a single vector (the conv bias) -> constant video term for text-only prompts (SURVEY App. A.9)
__global__ void ln_vector_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                 int d, float* __restrict__ y) {
  __shared__ float red[32];
  float s = 0.f;
  for (int c = threadIdx.x; c < d; c += blockDim.x) s += x[c];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) tot += red[i];
  const float mean = tot / (float)d;
  __syncthreads();
  float q = 0.f;
  for (int c = threadIdx.x; c < d; c += blockDim.x) { const float u = x[c] - mean; q += u * u; }
  q = warp_sum(q);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
  __syncthreads();
  float qt = 0.f;
  for (int i = 0; i < (int)(blockDim.x >> 5); ++i) qt += red[i];
  const float rstd = rsqrtf(qt / (float)d + 1e-5f);
  for (int c = threadIdx.x; c < d; c += blockDim.x) y[c] = (x[c] - mean) * rstd * w[c] + b[c];
}

// small dense fp32 product for load-time tables: C[i,j] = sum_k A[i,k] * B[j,k]   (anchor table 4 x d)
__global__ void small_abt_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C,
                                 int I, int J, int K) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= I * J) return;
  const int i = idx / J, j = idx % J;
  float s = 0.f;
  for (int k = 0; k < K; ++k) s = fmaf(A[i * K + k], B[(long long)j * K + k], s);
  C[idx] = s;
}

// RoPE table (rope.py:116-145): rope[pos][i] = (cos, sin)(pos * theta^(-2i/hd)), i < hd/2
__global__ void rope_table_kernel(float2* __restrict__ rope, int T, int hd, float theta) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= T * (hd / 2)) return;
  const int pos = idx / (hd / 2), i = idx % (hd / 2);
  const float inv = 1.0f / powf(theta, (float)(2 * i) / (float)hd);
  const float a = (float)pos * inv;
  rope[idx] = make_float2(cosf(a), sinf(a));
}

}  // namespace sab
