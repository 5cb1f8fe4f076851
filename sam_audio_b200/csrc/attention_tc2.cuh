// wgmma self-attention for sequences of up to 256 keys (10 s clips: T = 250), head_dim = 128.
// reference: sam_audio/model/transformer.py:153-160 (SDPA, scale 1/sqrt(hd), bool key mask, True = attend).
//
// One CTA per (item, head): TMA brings Q (one or two 128-query tiles), K and V ([256 x 128] each, SWIZZLE_128B,
// zero-filled past the sequence end) into shared memory once; two consumer warpgroups own 64 query rows each and
// walk the query tiles.  Everything between the two HBM touches stays on chip, the scores in registers:
//   wgmma : S = Q K^T            (m64n256k16 x 8, both operands from shared memory) -> 128 fp32 registers / thread
//   CUDA  : row softmax on the accumulator fragment (a row lives in the 4 lanes of a quad)
//   wgmma : O = P V              (m64n128k16 x 16, A = P as bf16 register fragments, B = V MN-major smem)
//   CUDA  : O / rowsum -> bf16 -> global, head-major "(h d)"
// Softmax variants: exact (two-pass row maximum), single pass with a per-layer bound `shift` >= every logit (with
// QK-RMSNorm, transformer.py:117-119,145-148: |q.k|/sqrt(hd) <= sqrt(hd) max|w_q| max|w_k|; softmax is
// shift-invariant), and `folded`, where the engine's QKV epilogue has already scaled q into the log2 domain and the
// bound is small enough (<= 50) that p = 2^s needs neither scale nor shift.  kPoly of every 8 exponential pairs run
// on the FMA pipe (Cody-Waite range reduction + degree-3 minimax polynomial, rel. error 7.5e-5, far below bf16's
// 3.9e-3), the rest on the MUFU.
// Longer sequences use the wgmma streaming kernel in attention_stream_tc.cuh.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace sab {

constexpr int AT2_THREADS = 256;                  // two consumer warpgroups
constexpr int AT2_Q_BYTES = 128 * 128 * 2;        // 32 KB per 128-query tile (2 boxes of [128 x 64])
constexpr int AT2_KV_BYTES = 256 * 128 * 2;       // 64 KB (2 boxes of [256 x 64])
constexpr int AT2_SMEM = 2 * AT2_Q_BYTES + 2 * AT2_KV_BYTES + 256 /*key validity*/ + 64 /*barriers*/ + 1024 /*alignment*/;
static_assert(AT2_SMEM <= 227 * 1024, "attention_tc2: shared memory budget");

struct AttnTc2Params {
  __nv_bfloat16* o; long long o_ld; // output [items * T, o_ld], head h at columns [128h, 128h + 128)
  const uint8_t* key_mask;          // [items / mask_div, Tk] or null
  int T, heads, items;
  int mask_div;                     // mask row = item / mask_div (candidates share their clip's pad mask); 0/1: item
  int q_col0, k_col0, v_col0;       // column of head 0 inside the fused QKV row
  float scale_log2;                 // log2(e) / sqrt(hd)
  float shift_log2;                 // single-pass variant: a bound on every scaled logit (log2 domain)
  int reverse;                      // walk the items from the last to the first (serpentine L2 reuse, engine.cu)
};

SAB_DEVICE float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// 2^x on the FMA / ALU pipes: n = rint(x), f = x - n in [-1/2, 1/2], 2^f by a degree-3 minimax polynomial
// (relative error 7.5e-5), 2^n by adding n to the exponent field
SAB_DEVICE float exp2_poly(float x) {
  constexpr float kMagic = 12582912.f;   // 1.5 * 2^23: adding it rounds to the nearest integer
  x = fmaxf(x, -125.f);
  const float t = __fadd_rn(x, kMagic);
  const float n = __fadd_rn(t, -kMagic);
  const float f = __fadd_rn(x, -n);
  float p = fmaf(0.0551716648f, f, 0.2426111251f);
  p = fmaf(p, f, 0.6932609677f);
  p = fmaf(p, f, 0.9999280572f);
  return __int_as_float(__float_as_int(p) + (__float_as_int(t) << 23));
}
template <bool kExact, int kPoly, bool kFolded>
__global__ void __launch_bounds__(AT2_THREADS, 1)
attention_tc2_kernel(const __grid_constant__ CUtensorMap tm_q /*box 64 x 128*/,
                     const __grid_constant__ CUtensorMap tm_k /*box 64 x 256*/,
                     const __grid_constant__ CUtensorMap tm_v /*box 64 x 256*/,
                     const __grid_constant__ AttnTc2Params P) {
  extern __shared__ uint8_t at2_raw[];
  uint8_t* at2_smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at2_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = at2_smem;                          // two query tiles
  uint8_t* sK = sQ + 2 * AT2_Q_BYTES;
  uint8_t* sV = sK + AT2_KV_BYTES;
  uint8_t* s_valid = sV + AT2_KV_BYTES;            // [256] key < T and not masked
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_valid + 256);
  uint64_t *bar_qk0 = bars, *bar_q1 = bars + 1, *bar_v = bars + 2;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wg = warp >> 2;                        // consumer warpgroup: query rows 64 wg .. 64 wg + 63 of a tile
  const int n_mt = (P.T + 127) / 128;              // 1 or 2 query tiles
  const int w = blockIdx.x;
  const int head = w % P.heads, item = P.reverse ? P.items - 1 - w / P.heads : w / P.heads;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    mbar_init(bar_qk0, 1);
    mbar_init(bar_q1, 1);
    mbar_init(bar_v, 1);
    fence_barrier_init();
  }
  {
    const uint8_t* mk = P.key_mask ? P.key_mask + (long long)(P.mask_div > 1 ? item / P.mask_div : item) * P.T : nullptr;
    const int key = threadIdx.x;
    s_valid[key] = (key < P.T && (!mk || mk[key])) ? 1 : 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int qc = P.q_col0 + head * 128, kc = P.k_col0 + head * 128, vc = P.v_col0 + head * 128;
    mbar_expect_tx(bar_qk0, AT2_Q_BYTES + AT2_KV_BYTES);
    tma_load_3d(sQ, &tm_q, bar_qk0, qc, 0, item);
    tma_load_3d(sQ + AT2_Q_BYTES / 2, &tm_q, bar_qk0, qc + 64, 0, item);
    tma_load_3d(sK, &tm_k, bar_qk0, kc, 0, item);
    tma_load_3d(sK + AT2_KV_BYTES / 2, &tm_k, bar_qk0, kc + 64, 0, item);
    if (n_mt > 1) {
      mbar_expect_tx(bar_q1, AT2_Q_BYTES);
      tma_load_3d(sQ + AT2_Q_BYTES, &tm_q, bar_q1, qc, 128, item);
      tma_load_3d(sQ + AT2_Q_BYTES + AT2_Q_BYTES / 2, &tm_q, bar_q1, qc + 64, 128, item);
    }
    mbar_expect_tx(bar_v, AT2_KV_BYTES);
    tma_load_3d(sV, &tm_v, bar_v, vc, 0, item);
    tma_load_3d(sV + AT2_KV_BYTES / 2, &tm_v, bar_v, vc + 64, 0, item);
  }

  // accumulator fragment: this thread holds rows r0 and r0 + 8 of the warpgroup's 64, columns 8i + 2 (lane % 4) + {0, 1}
  const int r0 = (warp & 3) * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  const float scale = kFolded ? 1.f : P.scale_log2;
  for (int m = 0; m < n_mt; ++m) {
    mbar_wait(m == 0 ? bar_qk0 : bar_q1, 0);
    // ---- S = Q K^T ----
    float s[128];
#pragma unroll
    for (int i = 0; i < 128; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t qa = smem_u32(sQ) + m * AT2_Q_BYTES + (ks >> 2) * (AT2_Q_BYTES / 2) + wg * 64 * 128;
      const uint32_t ka = smem_u32(sK) + (ks >> 2) * (AT2_KV_BYTES / 2);
      Wgmma<256>::ss(s, make_kmajor_desc<128>(qa) + (uint64_t)((ks & 3) * 2), make_kmajor_desc<128>(ka) + (uint64_t)((ks & 3) * 2), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // ---- softmax over the fragment: s[4i + 2h + j] = (row r0 + 8h, key 8i + c0 + j) ----
    float nshift[2] = {kFolded ? 0.f : -P.shift_log2, kFolded ? 0.f : -P.shift_log2};
    if constexpr (kExact) {
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 32; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
          if (s_valid[8 * i + c0 + j]) {
            mx[0] = fmaxf(mx[0], s[4 * i + j]);
            mx[1] = fmaxf(mx[1], s[4 * i + 2 + j]);
          }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
        mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
        nshift[h] = (mx[h] == -INFINITY) ? 0.f : -mx[h] * scale;
      }
    }
    float sum[2] = {0.f, 0.f};
    uint32_t pk[64];   // P as bf16 pairs, already in the A-fragment order of the PV wgmma
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const bool v0 = s_valid[8 * i + c0] != 0, v1 = s_valid[8 * i + c0 + 1] != 0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float x0 = kFolded ? s[4 * i + 2 * h] : fmaf(s[4 * i + 2 * h], scale, nshift[h]);
        const float x1 = kFolded ? s[4 * i + 2 * h + 1] : fmaf(s[4 * i + 2 * h + 1], scale, nshift[h]);
        float p0, p1;
        if (((2 * i + h) & 7) < kPoly) { p0 = exp2_poly(x0); p1 = exp2_poly(x1); }
        else { p0 = ex2_approx(x0); p1 = ex2_approx(x1); }
        p0 = v0 ? p0 : 0.f;
        p1 = v1 ? p1 : 0.f;
        sum[h] += p0 + p1;
        pk[2 * i + h] = pack_bf16(p0, p1);
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
      sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
    }

    // ---- O = P V: A fragment of key step ks = pk[4ks .. 4ks+3] (rows r0 / r0+8, keys 16ks + c0 / 16ks + 8 + c0) ----
    mbar_wait(bar_v, 0);
    float o[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 16; ++ks) {
      const uint32_t a[4] = {pk[4 * ks], pk[4 * ks + 1], pk[4 * ks + 2], pk[4 * ks + 3]};
      const uint64_t vb = make_mnmajor_desc(smem_u32(sV) + ks * 16 * 128, (uint32_t)(AT2_KV_BYTES / 2), 1024u);
      wgmma_rs_n128_bmn(o, a, vb, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    reg_fence(pk);

    // ---- epilogue: O / rowsum -> bf16 -> global (rows >= T dropped) ----
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = m * 128 + wg * 64 + r0 + 8 * h;
      if (row >= P.T) continue;
      const float inv = 1.f / sum[h];
      __nv_bfloat16* dst = P.o + ((long long)item * P.T + row) * P.o_ld + head * 128 + c0;
#pragma unroll
      for (int i = 0; i < 16; ++i)
        *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
    }
  }
}

}  // namespace sab
