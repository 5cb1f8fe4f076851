// wgmma / TMA streaming self-attention for sequences of more than 256 keys (clips longer than 10 s), head_dim = 128.
// reference: sam_audio/model/transformer.py:153-160 (SDPA, scale 1/sqrt(hd), bool key mask, True = attend).
//
// One CTA per 128-query tile of one (item, head).  blockIdx.x = (item * heads + head) * n_qt + qt, so the query tiles
// of one (item, head) are launched next to each other and all but the first read its K and V from L2.
//   warp 0       : TMA producer.  Q once, then K and V in blocks of 128 keys (32 KB each, SWIZZLE_128B, zero-filled
//                  past the sequence end) through a ring of ATS_STAGES mbarrier-guarded stages.  It also writes each
//                  block's key validity (key < T and not padded) as 128 bits beside the stage.
//   warps 4..11  : two consumer warpgroups, 64 query rows each.  Per key block
//                    wgmma : S = Q K^T      (m64n128k16 x 8, both operands from shared memory) -> 64 fp32 registers
//                    CUDA  : p = 2^(s - m)  on the accumulator fragment, packed to bf16 A fragments
//                    wgmma : O += P V       (m64n128k16 x 8, A = P from registers, B = V MN-major from shared memory)
//                  and at the end O / rowsum -> bf16 -> global, head-major "(h d)".  The two warpgroups are not
//                  synchronised with each other, so one's exponentials run under the other's wgmma.
// Softmax variants (the same choice attention_tc2 makes from the layer's logit bound):
//   bounded : the engine's QKV epilogue has scaled q into the log2 domain and the QK-norm weights bound |s| by `shift`
//             <= 50.  p = 2^s needs no running maximum, so row sums and O simply accumulate over the key blocks in
//             fp32 and nothing is rescaled.  Range: a row sum over 10 000 < 2^14 keys is below 2^(50 + 14) = 2^64 and
//             O below that times max|v|, far from fp32's 2^128; the largest p of a row is at least 2^-50, a normal
//             fp32 and bf16 number, so the quotient O / rowsum keeps full relative precision.
//   exact   : running row maximum, O and the row sum rescaled by 2^(m_old - m_new) at every block.
// A block whose keys are all masked adds p = 0 everywhere (exact: the maximum stays where it was); an item with no
// valid key at all gets zeros; rows >= T of the last query tile are computed on zero-filled Q and not stored.
#pragma once
#include "attention_tc2.cuh"   // AttnTc2Params, exp2_poly, ex2_approx
#include "gemm_tc.cuh"         // setmaxnreg

namespace sab {

constexpr int ATS_THREADS = 384;                  // warp 0: TMA producer, warps 1..3 idle, warps 4..11: consumers
constexpr int ATS_BK = 128;                       // keys per block
constexpr int ATS_STAGES = 3;
constexpr int ATS_TILE_BYTES = 128 * 128 * 2;     // 32 KB: a Q tile, or one block of K or of V (2 boxes of [128 x 64])
constexpr int ATS_STAGE_BYTES = 2 * ATS_TILE_BYTES;   // K | V
constexpr int ATS_SMEM = ATS_TILE_BYTES + ATS_STAGES * ATS_STAGE_BYTES + ATS_STAGES * 16 /*key validity bits*/ +
                         64 /*barriers*/ + 1024 /*alignment*/;
static_assert(ATS_SMEM <= 227 * 1024, "attention_stream_tc: shared memory budget");
static_assert(2 * ATS_STAGES + 1 <= 8, "attention_stream_tc: barrier block");

template <bool kExact, int kPoly>
__global__ void __launch_bounds__(ATS_THREADS, 1)
attention_stream_tc_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                           const __grid_constant__ CUtensorMap tm_v /*all three: box 64 x 128*/,
                           const __grid_constant__ AttnTc2Params P) {
  extern __shared__ uint8_t ats_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ats_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sKV = sQ + ATS_TILE_BYTES;
  uint32_t* s_vbits = reinterpret_cast<uint32_t*>(sKV + ATS_STAGES * ATS_STAGE_BYTES);   // [stage][4]: bit k = key k valid
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(s_vbits + ATS_STAGES * 4);
  uint64_t* empty_bar = full_bar + ATS_STAGES;
  uint64_t* q_bar = empty_bar + ATS_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_qt = (P.T + 127) / 128;
  const int nkb = (P.T + ATS_BK - 1) / ATS_BK;
  const int qt = blockIdx.x % n_qt, ih = blockIdx.x / n_qt;
  const int head = ih % P.heads, item = P.reverse ? P.items - 1 - ih / P.heads : ih / P.heads;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
    for (int s = 0; s < ATS_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);     // lane 0 of every consumer warp
    }
    mbar_init(q_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer (warps 1..3 only give their registers back) =====================
    setmaxnreg_dec<40>();
    if (warp != 0) return;
    const int qc = P.q_col0 + head * 128, kc = P.k_col0 + head * 128, vc = P.v_col0 + head * 128;
    if (lane == 0) {
      mbar_expect_tx(q_bar, ATS_TILE_BYTES);
      tma_load_3d(sQ, &tm_q, q_bar, qc, qt * 128, item);
      tma_load_3d(sQ + ATS_TILE_BYTES / 2, &tm_q, q_bar, qc + 64, qt * 128, item);
    }
    const uint8_t* mk = P.key_mask ? P.key_mask + (long long)(P.mask_div > 1 ? item / P.mask_div : item) * P.T : nullptr;
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < nkb; ++kb) {
      const int key0 = kb * ATS_BK;
      uint32_t bits[4];
#pragma unroll
      for (int w = 0; w < 4; ++w) {
        const int key = key0 + 32 * w + lane;
        bits[w] = __ballot_sync(0xffffffffu, key < P.T && (!mk || mk[key]));
      }
      mbar_wait(&empty_bar[stage], phase ^ 1);
      if (lane == 0) {
        // ordered before the consumers' reads by the release of the arrive below and the acquire of their wait
        *reinterpret_cast<uint4*>(s_vbits + stage * 4) = make_uint4(bits[0], bits[1], bits[2], bits[3]);
        uint8_t* sK = sKV + stage * ATS_STAGE_BYTES;
        uint8_t* sV = sK + ATS_TILE_BYTES;
        mbar_expect_tx(&full_bar[stage], ATS_STAGE_BYTES);
        tma_load_3d(sK, &tm_k, &full_bar[stage], kc, key0, item);
        tma_load_3d(sK + ATS_TILE_BYTES / 2, &tm_k, &full_bar[stage], kc + 64, key0, item);
        tma_load_3d(sV, &tm_v, &full_bar[stage], vc, key0, item);
        tma_load_3d(sV + ATS_TILE_BYTES / 2, &tm_v, &full_bar[stage], vc + 64, key0, item);
      }
      __syncwarp();
      if (++stage == ATS_STAGES) { stage = 0; phase ^= 1; }
    }
    return;
  }

  // ===================== consumers =====================
  setmaxnreg_inc<232>();
  const int cw = warp - 4;
  const int wg = cw >> 2;                          // query rows 64 wg .. 64 wg + 63 of the tile
  // accumulator fragment: this thread holds rows r0 and r0 + 8 of the warpgroup's 64, columns 8i + c0 + {0, 1}
  const int r0 = (cw & 3) * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  const float scale = P.scale_log2;                // exact variant only (1 when q is already scaled)

  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  float sum[2] = {0.f, 0.f};                       // this thread's share of the row sums (quad-reduced at the end)
  float mx[2] = {-INFINITY, -INFINITY};            // exact: running row maximum (raw logits)

  mbar_wait(q_bar, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int kb = 0; kb < nkb; ++kb) {
    mbar_wait(&full_bar[stage], phase);
    const uint32_t sK = smem_u32(sKV + stage * ATS_STAGE_BYTES);
    const uint32_t sV = sK + ATS_TILE_BYTES;
    // ---- S = Q K^T ----
    float s[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t qa = smem_u32(sQ) + (ks >> 2) * (ATS_TILE_BYTES / 2) + wg * 64 * 128;
      const uint32_t ka = sK + (ks >> 2) * (ATS_TILE_BYTES / 2);
      Wgmma<128>::ss(s, make_kmajor_desc<128>(qa) + (uint64_t)((ks & 3) * 2), make_kmajor_desc<128>(ka) + (uint64_t)((ks & 3) * 2), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);

    // ---- softmax terms of this block: s[4i + 2h + j] = (row r0 + 8h, key 8i + c0 + j) ----
    const uint4 vb = *reinterpret_cast<const uint4*>(s_vbits + stage * 4);
    const uint32_t vw[4] = {vb.x >> c0, vb.y >> c0, vb.z >> c0, vb.w >> c0};   // bit 8 (i % 4) + j of word i / 4
    float nshift[2] = {0.f, 0.f};
    if constexpr (kExact) {
      float bm[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int j = 0; j < 2; ++j)
          if ((vw[i >> 2] >> (8 * (i & 3) + j)) & 1u) {
            bm[0] = fmaxf(bm[0], s[4 * i + j]);
            bm[1] = fmaxf(bm[1], s[4 * i + 2 + j]);
          }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        bm[h] = fmaxf(bm[h], __shfl_xor_sync(0xffffffffu, bm[h], 1));
        bm[h] = fmaxf(bm[h], __shfl_xor_sync(0xffffffffu, bm[h], 2));
        const float m_new = fmaxf(mx[h], bm[h]);
        const float m_use = (m_new == -INFINITY) ? 0.f : m_new;     // no valid key yet: every p of the block is 0
        const float alpha = ex2_approx((mx[h] - m_use) * scale);    // 2^-inf = 0 while the row had no valid key
        mx[h] = m_new;
        nshift[h] = -m_use * scale;
        sum[h] *= alpha;
#pragma unroll
        for (int i = 0; i < 16; ++i) { o[4 * i + 2 * h] *= alpha; o[4 * i + 2 * h + 1] *= alpha; }
      }
    }
    uint32_t pk[32];   // P as bf16 pairs, already in the A-fragment order of the PV wgmma
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const bool v0 = (vw[i >> 2] >> (8 * (i & 3))) & 1u, v1 = (vw[i >> 2] >> (8 * (i & 3) + 1)) & 1u;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float x0 = kExact ? fmaf(s[4 * i + 2 * h], scale, nshift[h]) : s[4 * i + 2 * h];
        const float x1 = kExact ? fmaf(s[4 * i + 2 * h + 1], scale, nshift[h]) : s[4 * i + 2 * h + 1];
        float p0, p1;
        if (((2 * i + h) & 7) < kPoly) { p0 = exp2_poly(x0); p1 = exp2_poly(x1); }
        else { p0 = ex2_approx(x0); p1 = ex2_approx(x1); }
        p0 = v0 ? p0 : 0.f;
        p1 = v1 ? p1 : 0.f;
        sum[h] += p0 + p1;
        pk[2 * i + h] = pack_bf16(p0, p1);
      }
    }

    // ---- O += P V: A fragment of key step ks = pk[4ks .. 4ks+3] (rows r0 / r0+8, keys 16ks + c0 / 16ks + 8 + c0) ----
    reg_fence(o);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const uint32_t a[4] = {pk[4 * ks], pk[4 * ks + 1], pk[4 * ks + 2], pk[4 * ks + 3]};
      const uint64_t vd = make_mnmajor_desc(sV + ks * 16 * 128, (uint32_t)(ATS_TILE_BYTES / 2), 1024u);
      wgmma_rs_n128_bmn(o, a, vd, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    reg_fence(pk);
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == ATS_STAGES) { stage = 0; phase ^= 1; }
  }

  // ---- epilogue: O / rowsum -> bf16 -> global (rows >= T dropped) ----
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
    sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
    const int row = qt * 128 + wg * 64 + r0 + 8 * h;
    if (row >= P.T) continue;
    const float inv = sum[h] > 0.f ? 1.f / sum[h] : 0.f;   // an item with no valid key at all: zeros, not 0 * inf
    __nv_bfloat16* dst = P.o + ((long long)item * P.T + row) * P.o_ld + head * 128 + c0;
#pragma unroll
    for (int i = 0; i < 16; ++i)
      *reinterpret_cast<uint32_t*>(dst + 8 * i) = pack_bf16(o[4 * i + 2 * h] * inv, o[4 * i + 2 * h + 1] * inv);
  }
}

}  // namespace sab
