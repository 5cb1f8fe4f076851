// Persistent, warp-specialised wgmma GEMM for sm_90a:   D[m, n] = sum_k A[m', k'] * B[n, k]
//
//  * A (activations, bf16, K-major rows) arrives through a 3-D TMA map (cols, rows-per-item, items);
//    the K loop is a short list of "runs" (row_shift, a_col, n k-blocks), so the same kernel serves
//    plain linears (1 run), dilated / strided Conv1d and ConvTranspose1d over channels-last audio
//    (one run per tap; TMA zero-fills rows that fall off either end of an item = the conv's padding).
//  * B (weights, bf16, [N, Ktot] K-major, packed at load time) arrives through a 2-D TMA map.
//  * Warp 0 is the TMA producer (a ring of mbarrier-guarded stages); warps 4..11 form two consumer
//    warpgroups.  Warpgroup g multiplies rows 64g .. 64g+63 of the 128 x BN tile with wgmma.mma_async
//    (m64nBNk16, both operands from shared memory, fp32 accumulators in registers, one k-block in flight),
//    then writes its accumulators into an fp32 [128 x BN] shared-memory tile (16-byte units XOR-swizzled
//    by row, conflict-free for both access patterns below).  The same eight warps run the epilogue from
//    that tile, two warps per 32-row quarter taking alternating 32-column chunks: a thread reads one row's
//    32 values, or a transposed 4-column x 8-row block so that every global access is row-contiguous
//    (8 lanes x 16 B = one full 128 B line per row).  The producer refills the stages with the next tile
//    while the epilogue runs.
//  * CG = 1: one CTA per 128 x BN tile.
//    CG = 2: a 2-CTA cluster per 256 x BN tile: each CTA stages its own 128 A rows and loads HALF of the B
//    tile, multicast into both CTAs' shared memory, so B's L2 -> SMEM traffic per SM halves.  A stage is
//    refilled only when the consumers of both CTAs have released it (remote mbarrier arrives).
//  * Tiles are rasterised in groups of `group_m` m-tiles that sweep n: the A panel of a group stays in L2.
//  * Epilogues (fused, no extra pass over HBM):
//      EPI_AFFINE : v = (acc + bias[n]) * gate[row/gate_div, n] * alpha + res[row, n]
//                   -> fp32 and/or bf16 and/or Snake(v) bf16   (DiT residual/gate, ODE axpy, codec convs)
//      EPI_SWIGLU : silu(gate_cols) * up_cols -> bf16          (w1|w3 interleaved in 32-col chunks)
//      EPI_QKV    : per-head RMSNorm (q,k) + RoPE on adjacent pairs -> bf16   (heads are 128 contiguous cols)
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace sab {

constexpr int GEMM_BM = 128;
constexpr int GEMM_THREADS = 384;   // warp 0: TMA producer, warps 1..3 idle, warps 4..11: two consumer warpgroups
constexpr int GEMM_MAX_RUNS = 8;

// EPI_AFFINE_NORM = EPI_AFFINE + the producer half of the fused RMSNorm (own instantiation: the extra per-lane state
// would spill in the plain affine epilogue, which is already at the 168-register cap of a 384-thread CTA)
enum EpiMode { EPI_AFFINE = 0, EPI_SWIGLU = 1, EPI_QKV = 2, EPI_AFFINE_NORM = 3 };

struct KRun {
  int row_shift;  // added to the tile's first row (rows outside [0, rows_per_item) read as zero)
  int a_col;      // first A column (elements)
  int nkb;        // number of BK-wide k-blocks
};

struct GemmParams {
  // tiling
  int rows_per_item;    // T: rows per batch item (tiles never straddle items)
  int n_items;
  int tiles_per_item;   // ceil(T / (128 * CG))  — "unit" tiles (a CTA for CG=1, a CTA pair for CG=2)
  int N;                // valid output columns
  int n_tiles_n;
  int group_m;          // rasterisation: unit m-tiles per L2-resident A panel
  int reverse_m;        // walk the m-tiles from the last row block to the first (see engine.cu "serpentine")
  // K loop
  int n_runs[2];
  KRun runs[2][GEMM_MAX_RUNS];
  int n_period, n_switch;  // run list 1 iff n_period > 0 and (n0 % n_period) >= n_switch
  // affine epilogue
  const float* bias; int bias_mod;           // bias[n % bias_mod] (bias_mod == 0: bias[n])
  const float* gate; int gate_ld; int gate_div;
  float alpha;
  int relu;                                   // clamp at 0 after the residual add (T5 DenseReluDense)
  const float* res; long long res_ld;
  float* out_f32; long long out_f32_ld;
  __nv_bfloat16* out_bf16; long long out_bf16_ld;
  __nv_bfloat16* out_act; long long out_act_ld; const float* snake_alpha;  // snake_alpha[n % bias_mod]
  // fused RMSNorm + adaLN modulate (transformer.py:42-47,21-22), split between the producer of the residual stream and
  // the GEMM that consumes the normalised rows:  norm(h)*w*(1+scale)+shift  @ W^T
  //     =  rstd[row] * ((h * w*(1+scale)) @ W^T)  +  shift @ W^T
  //  producer (affine epilogue): out_scaled = bf16(v * colscale[row / gate_div][n]) is the consumer's A operand and
  //    ssq_out[row, 2*n_tile + warp_half] = sum of v^2 over the columns this epilogue warp owns (no atomics);
  //  consumer (every mode): acc' = rstd[row] * acc + ibias[row / ibias_div][n] before anything else,
  //    rstd[row] = rsqrt(sum_j ssq_in[row, j] * ssq_inv_dim + eps),  ibias = shift @ W^T (one small GEMM per evaluation)
  const float* colscale; long long colscale_ld;      // item = row / gate_div (as for the adaLN gate)
  __nv_bfloat16* out_scaled; long long out_scaled_ld;
  float* ssq_out; int ssq_ld;
  const float* ssq_in; int ssq_n; float ssq_inv_dim;
  const float* ibias; long long ibias_ld; int ibias_div;
  // back-to-back mode: acc1 = Snake_{b2b_alpha}(acc0 + b2b_bias) @ W1^T, then the affine epilogue runs on acc1
  const float* b2b_bias; const float* b2b_alpha;
  // qkv epilogue
  const float* qnorm_w; const float* knorm_w;  // [128]
  int n_q_end, n_k_end;                        // cols [0,n_q_end): q-norm, [n_q_end,n_k_end): k-norm, rest plain
  int qkv_period, norm_w_stride;               // > 0: the column pattern repeats every qkv_period columns (several layers'
                                               //      projections in one GEMM); repeat r uses norm weights + r*norm_w_stride
  const float2* rope; int rope_T; int use_rope; float eps;
  // fused cross-attention to a few text tokens (QKV mode, all heads are queries): instead of writing the normalised
  // queries, the epilogue attends to K/V [items*Tk, ld] (head-major columns; V at +xa_v_col0) and writes O
  const __nv_bfloat16* xa_kv; long long xa_kv_ld; int xa_v_col0; int xa_Tk;
  int xa_T;                 // query rows per K/V item (T x candidates: the candidates of a clip share its text K/V)
  const uint8_t* xa_mask;   // [items, Tk] or null
  float xa_scale_log2;
};
constexpr int XA_MAX_TK = 8;

template <int BN, int BK, int CG, bool B2B = false>
struct GemmSmem {
  static constexpr int kABytes = GEMM_BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kAccBytes = GEMM_BM * BN * 4;          // fp32 accumulator tile handed to the epilogue
  static constexpr int kBarBytes = 1024;
  // back-to-back second GEMM (1x1 conv of a residual unit): its [BN x BN] weight stays resident and the activated
  // 128 x BN intermediate tile is handed to the tensor core through shared memory, both K-major swizzled
  static constexpr int kW1Bytes = B2B ? BN * BN * 2 : 0;
  static constexpr int kMidBytes = B2B ? GEMM_BM * BN * 2 : 0;
  static constexpr int kBudget = 227 * 1024 - kAccBytes - kBarBytes - 1024 - kW1Bytes - kMidBytes;
  static constexpr int kStages = kBudget / kStageBytes > 8 ? 8 : kBudget / kStageBytes;
  static constexpr int kTotal = kStages * kStageBytes + kW1Bytes + kMidBytes + kAccBytes + kBarBytes + 1024;  // +1024: alignment
};

// ---- cluster helpers (CG = 2) ----
SAB_DEVICE uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
SAB_DEVICE void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster
SAB_DEVICE void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// TMA load written to the same offset in every CTA of `mask`; each destination CTA's mbarrier at `bar`'s offset
// receives the bytes it got
SAB_DEVICE void tma_load_2d_mc(void* smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
SAB_DEVICE void sts64(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}

// tile -> (unit m-tile, n-tile): groups of `group_m` m-tiles sweep n (m fastest inside a group)
SAB_DEVICE void tile_coords(int tile, int n_tiles_m, int n_tiles_n, int group_m, int reverse_m, int& mt, int& nt) {
  const int per_group = group_m * n_tiles_n;
  const int g = tile / per_group;
  const int idx = tile - g * per_group;
  const int m_first = g * group_m;
  const int gsz = (n_tiles_m - m_first < group_m) ? (n_tiles_m - m_first) : group_m;
  nt = idx / gsz;
  mt = m_first + (idx - nt * gsz);
  if (reverse_m) mt = n_tiles_m - 1 - mt;
}

SAB_DEVICE uint2 pack4_bf16(float4 v) { return make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w)); }

template <int BN, int BK, int MODE, int CG, bool B2B = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const __grid_constant__ CUtensorMap tmW /*B2B: [BN, BN] second weight, box BK x BN*/,
               const __grid_constant__ GemmParams P) {
  using S = GemmSmem<BN, BK, CG, B2B>;
  static_assert(!B2B || (CG == 1 && MODE == EPI_AFFINE && BN <= 128), "back-to-back mode: 1-CTA affine tiles, N <= 128");
  constexpr int kStages = S::kStages;
  static_assert(BN % 32 == 0 && BN >= 64 && BN <= 256, "invalid wgmma N / epilogue chunking");
  static_assert(BK == 64 || BK == 32, "BK must be one swizzle row (128B or 64B)");
  static_assert(CG == 1 || (CG == 2 && BN % 16 == 0), "cta group");
  static_assert(kStages >= 2, "pipeline too shallow");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_w1 = smem + kStages * S::kStageBytes;            // [BN/BK chunks][BN rows x BK] (B2B)
  uint8_t* s_mid = s_w1 + S::kW1Bytes;                         // [BN/BK chunks][128 rows x BK] (B2B)
  uint8_t* s_acc = s_mid + S::kMidBytes;                       // fp32 [128 x BN], swizzled
  uint8_t* bar_base = s_acc + S::kAccBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(bar_base);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* w1_bar = empty_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t cta_rank = (CG == 2) ? cluster_ctarank() : 0u;
  const int unit = blockIdx.x / CG, n_units = gridDim.x / CG;
  const int n_tiles_m = P.n_items * P.tiles_per_item;
  const int n_tiles = n_tiles_m * P.n_tiles_n;

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8 * CG);   // one arrive per consumer warp of every CTA that reads the stage's B
    }
    mbar_init(w1_bar, 1);
    fence_barrier_init();
  }
  if constexpr (CG == 2) cluster_sync_all(); else __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer (every CTA) =====================
    if (lane == 0) {
      if constexpr (B2B) {   // the second GEMM's weight: loaded once, resident for the CTA's lifetime
        mbar_expect_tx(w1_bar, S::kW1Bytes);
        for (int kc = 0; kc < BN / BK; ++kc) tma_load_2d(s_w1 + kc * (BN * BK * 2), &tmW, w1_bar, kc * BK, 0);
      }
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = unit; tile < n_tiles; tile += n_units) {
        int mt, nt;
        tile_coords(tile, n_tiles_m, P.n_tiles_n, P.group_m, P.reverse_m, mt, nt);
        const int item = mt / P.tiles_per_item;
        const int t0 = (mt % P.tiles_per_item) * (GEMM_BM * CG) + (int)cta_rank * GEMM_BM;
        const int n0 = nt * BN;
        const int nb = n0 + (int)cta_rank * (BN / CG);   // this CTA's slice of the B tile
        const int list = (P.n_period > 0 && (n0 % P.n_period) >= P.n_switch) ? 1 : 0;
        int kb_global = 0;
        for (int r = 0; r < P.n_runs[list]; ++r) {
          const KRun run = P.runs[list][r];
          for (int kb = 0; kb < run.nkb; ++kb, ++kb_global) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* sa = smem + stage * S::kStageBytes;
            uint8_t* sb = sa + S::kABytes;
            mbar_expect_tx(&full_bar[stage], S::kStageBytes);
            tma_load_3d(sa, &tmA, &full_bar[stage], run.a_col + kb * BK, t0 + run.row_shift, item);
            if constexpr (CG == 2)
              tma_load_2d_mc(sb + cta_rank * (BN / 2) * BK * 2, &tmB, &full_bar[stage], kb_global * BK, nb, (uint16_t)3);
            else
              tma_load_2d(sb, &tmB, &full_bar[stage], kb_global * BK, nb);
            if (++stage == kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: wgmma main loop, then the epilogue (8 warps, 2 per 32-row quarter) =====================
    const int e = warp - 4;                    // 0..7
    const int q = e & 3;                       // 32-row quarter of the tile this warp's epilogue covers
    const int half = e >> 2;                   // which alternating 32-column chunks this warp owns
    const int wg = e >> 2;                     // consumer warpgroup: wgmma rows 64 wg .. 64 wg + 63
    const int tr_r = lane >> 3;                // transposed mapping: pass p covers row 4p + tr_r,
    const int tr_c = (lane & 7) * 4;           //   4 consecutive columns tr_c .. tr_c+3
    const uint32_t acc_base = smem_u32(s_acc);
    const int arow = q * 32 + lane;            // this thread's row in the row-per-thread epilogue form
    // byte address of (row, col) in the accumulator tile: 16-byte unit (col / 4) XOR (row % 8)
    auto acc_addr = [&](int r, int col) -> uint32_t {
      return acc_base + (uint32_t)(r * BN * 4) + (uint32_t)((((col >> 2) ^ (r & 7))) << 4) + (uint32_t)((col & 3) * 4);
    };
    // 32 consecutive columns c .. c+31 of this thread's row
    auto acc_ld32 = [&](int c, float (&v)[32]) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float4 t = lds128(acc_addr(arow, c + 4 * j));
        v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
      }
    };
    // overwrite them (values derived from this thread's own row, read back transposed below)
    auto acc_put = [&](int c, const float (&v)[32]) {
#pragma unroll
      for (int j = 0; j < 8; ++j) sts128(acc_addr(arow, c + 4 * j), make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]));
      __syncwarp();
    };
    // transposed read of the warp's 32 x 32 block at column c: pass p = row q*32 + 4p + tr_r, columns c + tr_c .. +3
    auto acc_get = [&](int c, float4 (&x)[8]) {
#pragma unroll
      for (int p = 0; p < 8; ++p) x[p] = lds128(acc_addr(q * 32 + 4 * p + tr_r, c + tr_c));
    };
    float accr[BN / 2];
    // this warpgroup's accumulator fragment -> the shared tile (rows 64 wg + 16 (warp % 4) + lane / 4 [+ 8])
    auto acc_dump = [&]() {
      const int r0 = wg * 64 + (e & 3) * 16 + (lane >> 2);
#pragma unroll
      for (int i = 0; i < BN / 8; ++i) {
        const int col = 8 * i + 2 * (lane & 3);
        sts64(acc_addr(r0, col), accr[4 * i], accr[4 * i + 1]);
        sts64(acc_addr(r0 + 8, col), accr[4 * i + 2], accr[4 * i + 3]);
      }
    };
    auto release = [&](int s) {
      if (lane == 0) {
        mbar_arrive(&empty_bar[s]);
        if constexpr (CG == 2) mbar_arrive_cluster(&empty_bar[s], cta_rank ^ 1u);
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = unit; tile < n_tiles; tile += n_units) {
      int mt, nt;
      tile_coords(tile, n_tiles_m, P.n_tiles_n, P.group_m, P.reverse_m, mt, nt);
      const int item = mt / P.tiles_per_item;
      const int t_base = (mt % P.tiles_per_item) * (GEMM_BM * CG) + (int)cta_rank * GEMM_BM + q * 32;  // row of lane 0
      const long long row0 = (long long)item * P.rows_per_item + t_base + tr_r;   // this lane's row in pass 0
      const int rl = P.rows_per_item - t_base - tr_r;   // pass p is valid iff 4p < rl
      const int n0 = nt * BN;

      // ---- main loop: one k-block of wgmma in flight; a stage is released once the wgmma reading it retired ----
      {
        const int list = (P.n_period > 0 && (n0 % P.n_period) >= P.n_switch) ? 1 : 0;
        int total_kb = 0;
        for (int r = 0; r < P.n_runs[list]; ++r) total_kb += P.runs[list][r].nkb;
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) accr[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < total_kb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * S::kStageBytes);
          const uint64_t da = make_kmajor_desc<BK * 2>(sa + (uint32_t)(wg * 64 * BK * 2));
          const uint64_t db = make_kmajor_desc<BK * 2>(sa + S::kABytes);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < BK / 16; ++k) Wgmma<BN>::ss(accr, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), 1u);
          wgmma_commit();
          wgmma_wait<1>();
          reg_fence(accr);
          if (prev >= 0) release(prev);
          prev = stage;
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        reg_fence(accr);
        if (prev >= 0) release(prev);
      }
      acc_dump();
      named_bar_sync(1, 256);

      // fused-RMSNorm consumer: rstd and the per-item bias row of THIS LANE'S row (thread == row form); the loads are
      // issued before the accumulator wait
      float nrm_rstd = 1.f;
      const float* nrm_brow = nullptr;
      if (P.ssq_in != nullptr) {
        const int t_thr = t_base + lane;
        const long long grow = (long long)item * P.rows_per_item + (t_thr < P.rows_per_item ? t_thr : P.rows_per_item - 1);
        const float* sp = P.ssq_in + grow * P.ssq_n;
        float ssum = 0.f;
        for (int jj = 0; jj < P.ssq_n; ++jj) ssum += __ldg(sp + jj);
        nrm_rstd = rsqrtf(ssum * P.ssq_inv_dim + P.eps);
        nrm_brow = P.ibias + (long long)((uint32_t)grow / (uint32_t)P.ibias_div) * P.ibias_ld + n0;
      }

      constexpr bool kNorm = (MODE == EPI_AFFINE_NORM);
      if constexpr (MODE == EPI_AFFINE || MODE == EPI_AFFINE_NORM) {
        // fp32 residual rows are fetched one chunk ahead (8 independent 16 B loads per lane in flight while the
        // previous chunk is transposed and stored); the first chunk's loads go out before the accumulator wait.
        const float* res0 = P.res ? P.res + row0 * P.res_ld + n0 + tr_c : nullptr;
        const long long res_step = 4 * P.res_ld;
        float4 rr[8], rr_n[8];
        auto load_res = [&](int c, float4 (&r4)[8]) {
#pragma unroll
          for (int p = 0; p < 8; ++p) {
            r4[p] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (res0 && 4 * p < rl && n0 + c < P.N) r4[p] = ldg_stream128(res0 + p * res_step + c);
          }
        };
        // item (= row / gate_div) of each pass: indexes the adaLN gate rows and the fused-RMSNorm column-scale rows
        // (one integer division per pass and tile, not per chunk)
        int item_p[8];
        if (!B2B && (P.gate || (kNorm && P.out_scaled))) {
#pragma unroll
          for (int p = 0; p < 8; ++p)
            item_p[p] = (4 * p < rl) ? (int)((uint32_t)(row0 + 4 * p) / (uint32_t)P.gate_div) : 0;
        }
        float ssq[8];   // fused RMSNorm, producer side: running sum of squares of this warp's columns, per pass
        if constexpr (kNorm) {
#pragma unroll
          for (int p = 0; p < 8; ++p) ssq[p] = 0.f;
        }
        if constexpr (B2B) {
          // ---- first epilogue: Snake(acc0 + bias) -> bf16 -> the K-major swizzled A tile of the second GEMM ----
          const int r_tile = q * 32 + lane;                    // row of this thread inside the 128-row tile
#pragma unroll 1
          for (int c = half * 32; c < BN; c += 64) {
            float v[32];
            acc_ld32(c, v);
            uint32_t pk[16];
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 b4 = __ldg(reinterpret_cast<const float4*>(P.b2b_bias + c + j));
              const float4 a4 = __ldg(reinterpret_cast<const float4*>(P.b2b_alpha + c + j));
              float x0 = v[j] + b4.x, x1 = v[j + 1] + b4.y, x2 = v[j + 2] + b4.z, x3 = v[j + 3] + b4.w, sn;
              sn = __sinf(a4.x * x0); x0 = fmaf(sn * sn, rcp_approx(a4.x + 1e-9f), x0);
              sn = __sinf(a4.y * x1); x1 = fmaf(sn * sn, rcp_approx(a4.y + 1e-9f), x1);
              sn = __sinf(a4.z * x2); x2 = fmaf(sn * sn, rcp_approx(a4.z + 1e-9f), x2);
              sn = __sinf(a4.w * x3); x3 = fmaf(sn * sn, rcp_approx(a4.w + 1e-9f), x3);
              pk[j >> 1] = pack_bf16(x0, x1);
              pk[(j >> 1) + 1] = pack_bf16(x2, x3);
            }
            // chunk of BK columns kc, 16-byte unit u inside the row, XOR-swizzled like the TMA layout
            const uint32_t tile = smem_u32(s_mid) + (uint32_t)((c / BK) * (GEMM_BM * BK * 2) + r_tile * (BK * 2));
            const int u0 = (c % BK) / 8;
            const int sw = (BK == 64) ? (r_tile & 7) : ((r_tile >> 1) & 3);
#pragma unroll
            for (int u = 0; u < 4; ++u)
              sts128u(tile + (uint32_t)(((u0 + u) ^ sw) << 4), make_uint4(pk[4 * u], pk[4 * u + 1], pk[4 * u + 2], pk[4 * u + 3]));
          }
          fence_proxy_async();              // generic-proxy writes -> tensor core reads
          named_bar_sync(1, 256);           // intermediate tile complete; every warp is done with the first accumulators
          // ---- second GEMM: this warpgroup's 64 rows of the intermediate x the resident weight ----
          mbar_wait(w1_bar, 0);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) accr[i] = 0.f;
          wgmma_fence();
#pragma unroll
          for (int kc = 0; kc < BN / BK; ++kc) {
            const uint64_t dm = make_kmajor_desc<BK * 2>(smem_u32(s_mid + kc * (GEMM_BM * BK * 2) + wg * 64 * BK * 2));
            const uint64_t dw = make_kmajor_desc<BK * 2>(smem_u32(s_w1 + kc * (BN * BK * 2)));
#pragma unroll
            for (int k = 0; k < BK / 16; ++k) Wgmma<BN>::ss(accr, dm + (uint64_t)(k * 2), dw + (uint64_t)(k * 2), 1u);
          }
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(accr);
          acc_dump();
          named_bar_sync(1, 256);
          load_res(half * 32, rr);
        } else {
          load_res(half * 32, rr);
        }
#pragma unroll 1
        for (int c = half * 32; c < BN; c += 64) {
          if (n0 + c >= P.N) break;
          if (c + 64 < BN) load_res(c + 64, rr_n);
          const int n = n0 + c + tr_c;
          float4 g4[8];                         // gate values: requested before the accumulator read, used after
          if (!B2B && !kNorm && P.gate) {       // (the codec's back-to-back tiles have no gate: keep their registers)
            const float* g0 = P.gate + n;
#pragma unroll
            for (int p = 0; p < 8; ++p) g4[p] = __ldg(reinterpret_cast<const float4*>(g0 + item_p[p] * P.gate_ld));
          }
          float4 x[8];
          acc_get(c, x);
          if (P.bias) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(P.bias + (P.bias_mod ? (n % P.bias_mod) : n)));
#pragma unroll
            for (int p = 0; p < 8; ++p) { x[p].x += b4.x; x[p].y += b4.y; x[p].z += b4.z; x[p].w += b4.w; }
          }
          if (!B2B && !kNorm && P.gate) {
#pragma unroll
            for (int p = 0; p < 8; ++p) { x[p].x *= g4[p].x; x[p].y *= g4[p].y; x[p].z *= g4[p].z; x[p].w *= g4[p].w; }
          }
          if (kNorm && P.gate) {                // norm-producer instantiation: gate rows fetched at their use (L1/L2 hits)
            const float* g0 = P.gate + n;
#pragma unroll
            for (int p = 0; p < 8; ++p) {
              const float4 g = __ldg(reinterpret_cast<const float4*>(g0 + item_p[p] * P.gate_ld));
              x[p].x *= g.x; x[p].y *= g.y; x[p].z *= g.z; x[p].w *= g.w;
            }
          }
#pragma unroll
          for (int p = 0; p < 8; ++p) {
            x[p].x = fmaf(x[p].x, P.alpha, rr[p].x); x[p].y = fmaf(x[p].y, P.alpha, rr[p].y);
            x[p].z = fmaf(x[p].z, P.alpha, rr[p].z); x[p].w = fmaf(x[p].w, P.alpha, rr[p].w);
          }
          if (P.relu) {
#pragma unroll
            for (int p = 0; p < 8; ++p) {
              x[p].x = fmaxf(x[p].x, 0.f); x[p].y = fmaxf(x[p].y, 0.f); x[p].z = fmaxf(x[p].z, 0.f); x[p].w = fmaxf(x[p].w, 0.f);
            }
          }
          if (P.out_f32) {
            float* o0 = P.out_f32 + row0 * P.out_f32_ld + n;
            const long long st = 4 * P.out_f32_ld;
#pragma unroll
            for (int p = 0; p < 8; ++p)
              if (4 * p < rl) *reinterpret_cast<float4*>(o0 + p * st) = x[p];
          }
          if (P.out_bf16) {
            __nv_bfloat16* o0 = P.out_bf16 + row0 * P.out_bf16_ld + n;
            const long long st = 4 * P.out_bf16_ld;
#pragma unroll
            for (int p = 0; p < 8; ++p)
              if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
          }
          if (kNorm && P.out_scaled) {   // the next GEMM's A operand: h * w_norm * (1 + scale); and sum h^2
            __nv_bfloat16* o0 = P.out_scaled + row0 * P.out_scaled_ld + n;
            const long long st = 4 * P.out_scaled_ld;
            const float* c0 = P.colscale + n;
#pragma unroll
            for (int p = 0; p < 8; ++p) {
              const float4 c4 = __ldg(reinterpret_cast<const float4*>(c0 + item_p[p] * P.colscale_ld));
              ssq[p] = fmaf(x[p].x, x[p].x, fmaf(x[p].y, x[p].y, fmaf(x[p].z, x[p].z, fmaf(x[p].w, x[p].w, ssq[p]))));
              if (4 * p < rl)
                *reinterpret_cast<uint2*>(o0 + p * st) =
                    pack4_bf16(make_float4(x[p].x * c4.x, x[p].y * c4.y, x[p].z * c4.z, x[p].w * c4.w));
            }
          }
          if (P.out_act) {   // Snake: v + sin^2(a v) / (a + 1e-9)
            const float4 a4 = __ldg(reinterpret_cast<const float4*>(P.snake_alpha + (P.bias_mod ? (n % P.bias_mod) : n)));
            const float4 i4 = make_float4(rcp_approx(a4.x + 1e-9f), rcp_approx(a4.y + 1e-9f), rcp_approx(a4.z + 1e-9f), rcp_approx(a4.w + 1e-9f));
            __nv_bfloat16* o0 = P.out_act + row0 * P.out_act_ld + n;
            const long long st = 4 * P.out_act_ld;
#pragma unroll
            for (int p = 0; p < 8; ++p) {
              float s;
              s = __sinf(a4.x * x[p].x); x[p].x = fmaf(s * s, i4.x, x[p].x);
              s = __sinf(a4.y * x[p].y); x[p].y = fmaf(s * s, i4.y, x[p].y);
              s = __sinf(a4.z * x[p].z); x[p].z = fmaf(s * s, i4.z, x[p].z);
              s = __sinf(a4.w * x[p].w); x[p].w = fmaf(s * s, i4.w, x[p].w);
            }
#pragma unroll
            for (int p = 0; p < 8; ++p)
              if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
          }
#pragma unroll
          for (int p = 0; p < 8; ++p) rr[p] = rr_n[p];
          __syncwarp();  // staging tile is rewritten by the next chunk
        }
        if (kNorm && P.ssq_out) {   // the 8 lanes of a row hold 4 columns each: one partial per (row, n-tile, warp half)
#pragma unroll
          for (int p = 0; p < 8; ++p) {
            float sv = ssq[p];
            sv += __shfl_xor_sync(0xffffffffu, sv, 1);
            sv += __shfl_xor_sync(0xffffffffu, sv, 2);
            sv += __shfl_xor_sync(0xffffffffu, sv, 4);
            if ((lane & 7) == 0 && 4 * p < rl) P.ssq_out[(row0 + 4 * p) * P.ssq_ld + nt * 2 + half] = sv;
          }
        }
      } else if constexpr (MODE == EPI_SWIGLU) {
        // tile columns: [32 gate | 32 up] pairs -> BN/2 outputs at column n0/2; this warp owns alternating pairs
#pragma unroll 1
        for (int c = half * 64; c < BN; c += 128) {
          if (n0 + c >= P.N) break;
          float g[32], u[32];
          acc_ld32(c, g);
          acc_ld32(c + 32, u);
          if (P.ssq_in) {   // fused RMSNorm: rstd * acc + (shift @ W^T) of this row's item (L1-broadcast loads)
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 bg = __ldg(reinterpret_cast<const float4*>(nrm_brow + c + j));
              const float4 bu = __ldg(reinterpret_cast<const float4*>(nrm_brow + c + 32 + j));
              g[j] = fmaf(g[j], nrm_rstd, bg.x); g[j + 1] = fmaf(g[j + 1], nrm_rstd, bg.y);
              g[j + 2] = fmaf(g[j + 2], nrm_rstd, bg.z); g[j + 3] = fmaf(g[j + 3], nrm_rstd, bg.w);
              u[j] = fmaf(u[j], nrm_rstd, bu.x); u[j + 1] = fmaf(u[j + 1], nrm_rstd, bu.y);
              u[j + 2] = fmaf(u[j + 2], nrm_rstd, bu.z); u[j + 3] = fmaf(u[j + 3], nrm_rstd, bu.w);
            }
          }
#pragma unroll
          for (int j = 0; j < 32; ++j) g[j] = silu_f(g[j]) * u[j];
          acc_put(c, g);
          float4 x[8];
          acc_get(c, x);
          __nv_bfloat16* o0 = P.out_bf16 + row0 * P.out_bf16_ld + ((n0 + c) >> 1) + tr_c;
          const long long st = 4 * P.out_bf16_ld;
#pragma unroll
          for (int p = 0; p < 8; ++p)
            if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
          __syncwarp();
        }
      } else {  // EPI_QKV: each 128-col group is one head; this warp owns heads half, half+2, ... (BN=256: one each)
        int pos[8];                             // RoPE position of each pass (one modulo per tile)
#pragma unroll
        for (int p = 0; p < 8; ++p) pos[p] = (int)(((uint32_t)row0 + 4u * p) % (uint32_t)P.rope_T);   // rows < 2^31: no 64-bit division
        constexpr int kHeadStep = (BN >= 256) ? 256 : 128;   // BN=128: both warps of a quarter share the single head
#pragma unroll 1
        for (int hc = (BN >= 256 ? half * 128 : 0); hc < BN; hc += kHeadStep) {
          const int nh = n0 + hc;
          if (nh >= P.N) break;
          const int rep = P.qkv_period > 0 ? nh / P.qkv_period : 0;
          const int nhp = P.qkv_period > 0 ? nh - rep * P.qkv_period : nh;
          const float* nw = (nhp < P.n_q_end) ? P.qnorm_w + rep * P.norm_w_stride
                                               : (nhp < P.n_k_end ? P.knorm_w + rep * P.norm_w_stride : nullptr);
          if (P.xa_kv != nullptr) {
            // ---- fused cross-attention (thread == query row; scores are linear in the un-normalised query) ----
            const int t_thr = t_base + lane;                                   // row inside the GEMM item
            const long long grow = (long long)item * P.rows_per_item + (t_thr < P.rows_per_item ? t_thr : P.rows_per_item - 1);
            const int b = (int)((uint32_t)grow / (uint32_t)P.xa_T);
            const __nv_bfloat16* kp = P.xa_kv + (long long)b * P.xa_Tk * P.xa_kv_ld + nh;
            const __nv_bfloat16* vp = kp + P.xa_v_col0;
            float ss = 0.f, sc[XA_MAX_TK];
#pragma unroll
            for (int j = 0; j < XA_MAX_TK; ++j) sc[j] = 0.f;
#pragma unroll 1
            for (int c = 0; c < 128; c += 32) {
              float v[32];
              acc_ld32(hc + c, v);
#pragma unroll
              for (int i = 0; i < 32; i += 4) {
                const float4 w4 = __ldg(reinterpret_cast<const float4*>(nw + c + i));
                ss = fmaf(v[i], v[i], ss); ss = fmaf(v[i + 1], v[i + 1], ss);
                ss = fmaf(v[i + 2], v[i + 2], ss); ss = fmaf(v[i + 3], v[i + 3], ss);
                v[i] *= w4.x; v[i + 1] *= w4.y; v[i + 2] *= w4.z; v[i + 3] *= w4.w;
              }
#pragma unroll
              for (int j = 0; j < XA_MAX_TK; ++j) {
                if (j < P.xa_Tk) {
                  const uint4* kr = reinterpret_cast<const uint4*>(kp + (long long)j * P.xa_kv_ld + c);
                  float d = 0.f;
#pragma unroll
                  for (int i = 0; i < 4; ++i) {
                    const uint4 k8 = __ldg(kr + i);
                    const float2 k0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&k8.x));
                    const float2 k1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&k8.y));
                    const float2 k2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&k8.z));
                    const float2 k3 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&k8.w));
                    d = fmaf(v[8 * i], k0.x, d); d = fmaf(v[8 * i + 1], k0.y, d);
                    d = fmaf(v[8 * i + 2], k1.x, d); d = fmaf(v[8 * i + 3], k1.y, d);
                    d = fmaf(v[8 * i + 4], k2.x, d); d = fmaf(v[8 * i + 5], k2.y, d);
                    d = fmaf(v[8 * i + 6], k3.x, d); d = fmaf(v[8 * i + 7], k3.y, d);
                  }
                  sc[j] += d;
                }
              }
            }
            const float rstd = rsqrtf(ss * (1.f / 128.f) + P.eps);
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < XA_MAX_TK; ++j) {
              const bool ok = j < P.xa_Tk && (!P.xa_mask || P.xa_mask[(long long)b * P.xa_Tk + j]);
              sc[j] = ok ? sc[j] * rstd * P.xa_scale_log2 : -INFINITY;
              mx = fmaxf(mx, sc[j]);
            }
            float den = 0.f;
#pragma unroll
            for (int j = 0; j < XA_MAX_TK; ++j) {
              float pj;
              asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(pj) : "f"(sc[j] - mx));
              sc[j] = pj;
              den += pj;
            }
            const float inv = 1.f / den;
#pragma unroll 1
            for (int c = 0; c < 128; c += 32) {
              float o[32];
#pragma unroll
              for (int i = 0; i < 32; ++i) o[i] = 0.f;
#pragma unroll
              for (int j = 0; j < XA_MAX_TK; ++j) {
                if (j < P.xa_Tk) {
                  const uint4* vr = reinterpret_cast<const uint4*>(vp + (long long)j * P.xa_kv_ld + c);
                  const float pj = sc[j] * inv;
#pragma unroll
                  for (int i = 0; i < 4; ++i) {
                    const uint4 v8 = __ldg(vr + i);
                    const float2 v0 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v8.x));
                    const float2 v1 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v8.y));
                    const float2 v2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v8.z));
                    const float2 v3 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v8.w));
                    o[8 * i] = fmaf(pj, v0.x, o[8 * i]); o[8 * i + 1] = fmaf(pj, v0.y, o[8 * i + 1]);
                    o[8 * i + 2] = fmaf(pj, v1.x, o[8 * i + 2]); o[8 * i + 3] = fmaf(pj, v1.y, o[8 * i + 3]);
                    o[8 * i + 4] = fmaf(pj, v2.x, o[8 * i + 4]); o[8 * i + 5] = fmaf(pj, v2.y, o[8 * i + 5]);
                    o[8 * i + 6] = fmaf(pj, v3.x, o[8 * i + 6]); o[8 * i + 7] = fmaf(pj, v3.y, o[8 * i + 7]);
                  }
                }
              }
              acc_put(hc + c, o);
              float4 x[8];
              acc_get(hc + c, x);
              __nv_bfloat16* o0 = P.out_bf16 + row0 * P.out_bf16_ld + nh + c + tr_c;
              const long long st = 4 * P.out_bf16_ld;
#pragma unroll
              for (int p = 0; p < 8; ++p)
                if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
              __syncwarp();
            }
            continue;
          }
          float rstd = 1.f;   // of this thread's row (lane = row)
          if (nw) {
            float ss = 0.f;
#pragma unroll 1
            for (int c = 0; c < 128; c += 32) {
              float v[32];
              acc_ld32(hc + c, v);
              if (P.ssq_in) {   // fused RMSNorm of the GEMM's input rows: the head's values are rstd * acc + bias
#pragma unroll
                for (int j = 0; j < 32; j += 4) {
                  const float4 b4 = __ldg(reinterpret_cast<const float4*>(nrm_brow + hc + c + j));
                  v[j] = fmaf(v[j], nrm_rstd, b4.x); v[j + 1] = fmaf(v[j + 1], nrm_rstd, b4.y);
                  v[j + 2] = fmaf(v[j + 2], nrm_rstd, b4.z); v[j + 3] = fmaf(v[j + 3], nrm_rstd, b4.w);
                }
              }
#pragma unroll
              for (int j = 0; j < 32; ++j) ss = fmaf(v[j], v[j], ss);
            }
            rstd = rsqrtf(ss * (1.f / 128.f) + P.eps);
          }
          float rs[8];
#pragma unroll
          for (int p = 0; p < 8; ++p) rs[p] = __shfl_sync(0xffffffffu, rstd, 4 * p + tr_r);
          float nrs[8];       // fused RMSNorm: rstd of each pass's row, and its item's bias row
          int nboff[8];
          if (P.ssq_in) {
#pragma unroll
            for (int p = 0; p < 8; ++p) {
              nrs[p] = __shfl_sync(0xffffffffu, nrm_rstd, 4 * p + tr_r);
              nboff[p] = (4 * p < rl) ? (int)((uint32_t)(row0 + 4 * p) / (uint32_t)P.ibias_div) * (int)P.ibias_ld : 0;
            }
          }
#pragma unroll 1
          for (int c = (BN >= 256 ? 0 : half * 32); c < 128; c += (BN >= 256 ? 32 : 64)) {
            const int cc = c + tr_c;              // column inside the head
            float4 x[8];
            acc_get(hc + c, x);
            if (P.ssq_in) {
              const float* b0 = P.ibias + nh + cc;
#pragma unroll
              for (int p = 0; p < 8; ++p) {
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(b0 + nboff[p]));
                x[p].x = fmaf(x[p].x, nrs[p], b4.x); x[p].y = fmaf(x[p].y, nrs[p], b4.y);
                x[p].z = fmaf(x[p].z, nrs[p], b4.z); x[p].w = fmaf(x[p].w, nrs[p], b4.w);
              }
            }
            if (nw) {
              const float4 w4 = __ldg(reinterpret_cast<const float4*>(nw + cc));
#pragma unroll
              for (int p = 0; p < 8; ++p) {
                x[p].x *= rs[p] * w4.x; x[p].y *= rs[p] * w4.y; x[p].z *= rs[p] * w4.z; x[p].w *= rs[p] * w4.w;
              }
              if (P.use_rope) {
#pragma unroll
                for (int p = 0; p < 8; ++p) {
                  const float4 cs = __ldg(reinterpret_cast<const float4*>(P.rope + (long long)pos[p] * 64 + (cc >> 1)));
                  const float a0 = x[p].x * cs.x - x[p].y * cs.y, a1 = x[p].x * cs.y + x[p].y * cs.x;
                  const float b0 = x[p].z * cs.z - x[p].w * cs.w, b1 = x[p].z * cs.w + x[p].w * cs.z;
                  x[p] = make_float4(a0, a1, b0, b1);
                }
              }
            }
            __nv_bfloat16* o0 = P.out_bf16 + row0 * P.out_bf16_ld + nh + cc;
            const long long st = 4 * P.out_bf16_ld;
#pragma unroll
            for (int p = 0; p < 8; ++p)
              if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
            __syncwarp();
          }
        }
      }
      named_bar_sync(1, 256);   // the accumulator tile may be overwritten by the next tile's main loop
    }
  }

  if constexpr (CG == 2) cluster_sync_all(); else __syncthreads();
}

}  // namespace sab
