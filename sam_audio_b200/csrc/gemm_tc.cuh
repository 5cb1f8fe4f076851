// Persistent, warp-specialised wgmma GEMM for sm_90a:   D[m, n] = sum_k A[m', k'] * B[n, k]
//
//  * A (activations, bf16, K-major rows) arrives through a 3-D TMA map (cols, rows-per-item, items);
//    the K loop is a short list of "runs" (row_shift, a_col, n k-blocks), so the same kernel serves
//    plain linears (1 run), dilated / strided Conv1d and ConvTranspose1d over channels-last audio
//    (one run per tap; TMA zero-fills rows that fall off either end of an item = the conv's padding).
//  * B (weights, bf16, [N, Ktot] K-major, packed at load time) arrives through a 2-D TMA map.
//  * Warp 0 is the TMA producer (a ring of mbarrier-guarded stages; its warpgroup gives registers back with
//    setmaxnreg, 40 per thread, so that the consumers get 232); warps 4..11 form two consumer warpgroups.
//    Warpgroup g multiplies rows 64g .. 64g+63 of the 128 x BN tile with wgmma.mma_async (m64nBNk16, both
//    operands from shared memory, fp32 accumulators in registers, one k-block in flight).
//  * The epilogue runs from the accumulator registers: each consumer warp owns 16 rows x BN of the tile and
//    walks them in 32-column chunks.  Element-wise work that fits the fragment layout (SwiGLU pairs, the
//    back-to-back Snake, cross-attention P V) is done in registers; each chunk then passes through a 2 KB
//    per-warp staging block (16-byte units XOR-swizzled by row, conflict-free both ways) and is read back
//    transposed, 4 columns x 4 rows per lane, so that every global access is row-contiguous (8 lanes x 16 B =
//    one full 128 B line per fp32 row).  Per-row sums (QK-norm, cross-attention scores) read the staged chunk
//    in row form (lane = row) and keep their sequential column order.  Without an fp32 accumulator tile the
//    ring gets 4 stages at BN = 256, and the producer prefetches the next tile's first k-blocks while the
//    epilogue runs.
//  * CG = 1: one CTA per 128 x BN tile.
//    CG = 2: a 2-CTA cluster per 256 x BN tile: each CTA stages its own 128 A rows and loads HALF of the B
//    tile, multicast into both CTAs' shared memory, so B's L2 -> SMEM traffic per SM halves.  A stage is
//    refilled only when the consumers of both CTAs have released it (remote mbarrier arrives).
//  * Tiles are rasterised in groups of `group_m` m-tiles that sweep n: the A panel of a group stays in L2.
//  * Epilogues (fused, no extra pass over HBM):
//      EPI_AFFINE : v = (acc + bias[n]) * gate[row/gate_div, n] * alpha + res[row, n]
//                   -> fp32 and/or bf16 and/or Snake(v) bf16   (DiT residual/gate, ODE axpy, codec convs)
//      EPI_SWIGLU : silu(gate_cols) * up_cols -> bf16          (w1|w3 interleaved in 32-col chunks)
//      EPI_QKV    : per-head RMSNorm (q,k) + RoPE on adjacent pairs -> bf16   (heads are 128 contiguous cols);
//                   or attention to a few text tokens -> O, or (XAP) -> the probabilities only
//  * A per-clip B operand (b_clip_rows > 0) lets cross.wo multiply the probabilities with its clip's folded values.
#pragma once
#include "common.cuh"
#include "wgmma.cuh"

namespace sab {

constexpr int GEMM_BM = 128;
constexpr int GEMM_THREADS = 384;   // warp 0: TMA producer, warps 1..3 idle, warps 4..11: two consumer warpgroups
constexpr int GEMM_MAX_RUNS = 8;

// EPI_AFFINE_NORM = EPI_AFFINE + the producer half of the fused RMSNorm (own instantiation: the plain affine epilogue
// keeps the registers of the sum-of-squares state for its gate prefetch)
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
  //    ssq_out[row, 2*n_tile + parity] = sum of v^2 over the tile's even (parity 0) or odd 32-column chunks (no atomics);
  //  consumer (SwiGLU and QKV without fused cross-attention; the host rejects ssq_in elsewhere):
  //    acc' = rstd[row] * acc + ibias[row / ibias_div][n] before anything else,
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
  // ... or, with xa_p set (XAP instantiation), writes each row's normalised probabilities to xa_p[row, j * heads + head]
  // (bf16; masked tokens exactly 0; token-major, so that a token's column does not depend on Tk) and no O: the output
  // projection then runs as a per-clip GEMM over them (see b_clip_rows)
  __nv_bfloat16* xa_p; long long xa_p_ld;
  // per-clip B operand: item i multiplies rows (i / b_clip_div) * b_clip_rows + [0, N) of B (0: one B shared by all)
  int b_clip_rows, b_clip_div;
};
constexpr int XA_MAX_TK = 8;

template <int BN, int BK, int CG, bool B2B = false>
struct GemmSmem {
  static constexpr int kABytes = GEMM_BM * BK * 2;
  static constexpr int kBBytes = BN * BK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kWarpStageBytes = 16 * 32 * 4;          // one consumer warp's 16 x 32 fp32 epilogue staging block
  static constexpr int kEpiBytes = 8 * kWarpStageBytes;        // 16 KB for the 8 consumer warps
  static constexpr int kBarBytes = 1024;
  // back-to-back second GEMM (1x1 conv of a residual unit): its [BN x BN] weight stays resident and the activated
  // 128 x BN intermediate tile is handed to the tensor core through shared memory, both K-major swizzled
  static constexpr int kW1Bytes = B2B ? BN * BN * 2 : 0;
  static constexpr int kMidBytes = B2B ? GEMM_BM * BN * 2 : 0;
  static constexpr int kBudget = 227 * 1024 - kEpiBytes - kBarBytes - 1024 - kW1Bytes - kMidBytes;
  static constexpr int kStages = kBudget / kStageBytes > 8 ? 8 : kBudget / kStageBytes;
  static constexpr int kTotal = kStages * kStageBytes + kW1Bytes + kMidBytes + kEpiBytes + kBarBytes + 1024;  // +1024: alignment
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
// arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster.  Used to release a stage to the
// peer's producer: the only accesses to order before it are the reads of the stage by wgmma, and those have completed
// when wgmma.wait_group returned (before this arrive is issued), so the default (.release.cta) semantics suffice and
// no cluster- or GPU-scope fence is needed on the k-block path.
SAB_DEVICE void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(cta));
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(remote) : "memory");
}
// warpgroup-wide register re-allocation (every warp of the warpgroup executes the same instruction)
template <int kRegs> SAB_DEVICE void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs> SAB_DEVICE void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
SAB_DEVICE void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }
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

// XAP: the fused cross-attention writes probabilities (xa_p) instead of O (its own instantiation: the two epilogues
// together do not fit the consumer's registers)
template <int BN, int BK, int MODE, int CG, bool B2B = false, bool XAP = false>
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
  // with a 2-stage ring the TMA load of k-block kb+1 is issued only as k-block kb starts: the tensor core waits on memory
  static_assert(BN != 256 || kStages >= 4, "256-wide tiles need at least 4 pipeline stages");
  static_assert(MODE != EPI_SWIGLU || BN % 64 == 0, "SwiGLU tiles hold whole [32 gate | 32 up] column pairs");
  static_assert(MODE != EPI_QKV || BN % 128 == 0, "QKV tiles hold whole 128-column heads");
  static_assert(!XAP || MODE == EPI_QKV, "cross-attention probabilities come from the QKV epilogue");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_w1 = smem + kStages * S::kStageBytes;            // [BN/BK chunks][BN rows x BK] (B2B)
  uint8_t* s_mid = s_w1 + S::kW1Bytes;                         // [BN/BK chunks][128 rows x BK] (B2B)
  uint8_t* s_epi = s_mid + S::kMidBytes;                       // [8 consumer warps][16 x 32 fp32], swizzled
  uint8_t* bar_base = s_epi + S::kEpiBytes;
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

  if (warp < 4) {
    // ===================== TMA producer (warp 0 of every CTA; warps 1..3 only give their registers back) =====================
    setmaxnreg_dec<40>();
    if (warp == 0 && lane == 0) {
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
        // this CTA's slice of the B tile (of the item's clip, for a per-clip B: both CTAs of a cluster share the item)
        const int nb = n0 + (int)cta_rank * (BN / CG) + (P.b_clip_rows ? (item / P.b_clip_div) * P.b_clip_rows : 0);
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
  } else {
    // ===================== consumers: wgmma main loop, then the epilogue on the accumulator fragment =====================
    setmaxnreg_inc<232>();
    const int e = warp - 4;                    // 0..7: this warp owns rows 16e .. 16e+15 of the 128-row tile
    const int wg = e >> 2;                     // consumer warpgroup: wgmma rows 64 wg .. 64 wg + 63
    const int fr = lane >> 2;                  // fragment form: rows fr and fr + 8 of the warp's 16 rows,
    const int fc = 2 * (lane & 3);             //   columns 8i + fc, 8i + fc + 1 of every 8-column group i
    const int tr_r = lane >> 3;                // transposed form: pass p covers row 4p + tr_r,
    const int tr_c = (lane & 7) * 4;           //   4 consecutive columns tr_c .. tr_c+3 of a 32-column chunk
    const uint32_t epi_base = smem_u32(s_epi) + (uint32_t)(e * S::kWarpStageBytes);
    // byte address of (row r < 16, col < 32) in this warp's staging block: 16-byte unit (col / 4) XOR (r % 8), which
    // is conflict-free for both the fragment writes and the transposed reads
    auto epi_addr = [&](int r, int col) -> uint32_t {
      return epi_base + (uint32_t)(r * 128) + (uint32_t)((((col >> 2) ^ (r & 7))) << 4) + (uint32_t)((col & 3) * 4);
    };
    // one 32-column chunk of fragment values -> the staging block: f[4i .. 4i+3] = (row fr, cols 8i+fc, +1), (row fr+8, ...)
    auto frag_put = [&](const float* f) {
      __syncwarp();                            // the previous chunk's transposed reads are done
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        sts64(epi_addr(fr, 8 * i + fc), f[4 * i], f[4 * i + 1]);
        sts64(epi_addr(fr + 8, 8 * i + fc), f[4 * i + 2], f[4 * i + 3]);
      }
      __syncwarp();
    };
    // ... read back transposed, so that the 8 lanes of a row cover its 32 columns and every global access is
    // row-contiguous (128 B per row for fp32, 64 B for bf16)
    auto stage_get = [&](float4 (&x)[4]) {
#pragma unroll
      for (int p = 0; p < 4; ++p) x[p] = lds128(epi_addr(4 * p + tr_r, tr_c));
    };
    float accr[BN / 2];
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
      const int t_base = (mt % P.tiles_per_item) * (GEMM_BM * CG) + (int)cta_rank * GEMM_BM + e * 16;  // warp's first row
      const long long row0 = (long long)item * P.rows_per_item + t_base + tr_r;   // this lane's row in pass 0
      const int rl = P.rows_per_item - t_base - tr_r;   // pass p is valid iff 4p < rl
      const int n0 = nt * BN;
      // global row of the warp's row r (0..15), clamped into the item (for row-indexed side inputs)
      auto row_grow = [&](int r) -> long long {
        const int t = t_base + r;
        return (long long)item * P.rows_per_item + (t < P.rows_per_item ? t : P.rows_per_item - 1);
      };
      // fused-RMSNorm consumer: rstd and the per-item bias row (ibias) of the warp's row r
      auto nrm_row = [&](int r, float& rstd, const float*& brow) {
        const long long grow = row_grow(r);
        const float* sp = P.ssq_in + grow * P.ssq_n;
        float ssum = 0.f;
        for (int jj = 0; jj < P.ssq_n; ++jj) ssum += __ldg(sp + jj);
        rstd = rsqrtf(ssum * P.ssq_inv_dim + P.eps);
        brow = P.ibias + (long long)((uint32_t)grow / (uint32_t)P.ibias_div) * P.ibias_ld + n0;
      };

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


      constexpr bool kNorm = (MODE == EPI_AFFINE_NORM);
      if constexpr (MODE == EPI_AFFINE || MODE == EPI_AFFINE_NORM) {
        // fp32 residual rows are fetched one chunk ahead (4 independent 16 B loads per lane in flight while the
        // current chunk is finished and stored); the first chunk's loads go out before the first staging.
        const float* res0 = P.res ? P.res + row0 * P.res_ld + n0 + tr_c : nullptr;
        const long long res_step = 4 * P.res_ld;
        float4 rr[4], rr_n[4];
        auto load_res = [&](int c, float4 (&r4)[4]) {
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            r4[p] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (res0 && 4 * p < rl && n0 + c < P.N) r4[p] = ldg_stream128(res0 + p * res_step + c);
          }
        };
        // item (= row / gate_div) of each pass: indexes the adaLN gate rows and the fused-RMSNorm column-scale rows
        // (one integer division per pass and tile, not per chunk)
        int item_p[4];
        if (!B2B && (P.gate || (kNorm && P.out_scaled))) {
#pragma unroll
          for (int p = 0; p < 4; ++p)
            item_p[p] = (4 * p < rl) ? (int)((uint32_t)(row0 + 4 * p) / (uint32_t)P.gate_div) : 0;
        }
        // fused RMSNorm, producer side: running sum of squares per pass, kept apart for even and odd 32-column chunks
        // (two partials per row and n-tile, as the consumer's ssq_n expects)
        float ssq[2][4];
        if constexpr (kNorm) {
#pragma unroll
          for (int p = 0; p < 4; ++p) ssq[0][p] = ssq[1][p] = 0.f;
        }
        if constexpr (B2B) {
          // ---- first epilogue: Snake(acc0 + bias) -> bf16, from the fragment straight into the K-major swizzled A
          //      tile of the second GEMM (4 lanes of a row fill one 16-byte unit) ----
#pragma unroll
          for (int i = 0; i < BN / 8; ++i) {
            const int col = 8 * i + fc;
            const float2 b2 = __ldg(reinterpret_cast<const float2*>(P.b2b_bias + col));
            const float2 a2 = __ldg(reinterpret_cast<const float2*>(P.b2b_alpha + col));
            const uint32_t chunk = smem_u32(s_mid) + (uint32_t)((col / BK) * (GEMM_BM * BK * 2));
            const int u = (col % BK) / 8;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int r = e * 16 + fr + 8 * h;          // row inside the 128-row tile
              float x0 = accr[4 * i + 2 * h] + b2.x, x1 = accr[4 * i + 2 * h + 1] + b2.y, sn;
              sn = __sinf(a2.x * x0); x0 = fmaf(sn * sn, rcp_approx(a2.x + 1e-9f), x0);
              sn = __sinf(a2.y * x1); x1 = fmaf(sn * sn, rcp_approx(a2.y + 1e-9f), x1);
              const int sw = (BK == 64) ? (r & 7) : ((r >> 1) & 3);
              sts32(chunk + (uint32_t)(r * (BK * 2) + ((u ^ sw) << 4) + (col & 7) * 2), pack_bf16(x0, x1));
            }
          }
          fence_proxy_async();              // generic-proxy writes -> tensor core reads
          named_bar_sync(1 + wg, 128);      // this warpgroup's 64 rows of the intermediate tile are complete
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
          named_bar_sync(1 + wg, 128);      // no warp rewrites the intermediate tile (next tile) before the wgmma retired
        }
        load_res(0, rr);
#pragma unroll
        for (int c = 0; c < BN; c += 32) {
          if (n0 + c >= P.N) break;
          const int n = n0 + c + tr_c;
          float4 g4[4];                         // gate values: requested before the staging, used after
          if (!B2B && !kNorm && P.gate) {       // (the codec's back-to-back tiles have no gate: keep their registers)
            const float* g0 = P.gate + n;
#pragma unroll
            for (int p = 0; p < 4; ++p) g4[p] = __ldg(reinterpret_cast<const float4*>(g0 + item_p[p] * P.gate_ld));
          }
          float4 x[4];
          frag_put(&accr[c / 2]);
          stage_get(x);
          // next chunk's residual, issued once this chunk's accumulator registers are free
          if (c + 32 < BN) load_res(c + 32, rr_n);
          if (P.bias) {
            const float4 b4 = __ldg(reinterpret_cast<const float4*>(P.bias + (P.bias_mod ? (n % P.bias_mod) : n)));
#pragma unroll
            for (int p = 0; p < 4; ++p) { x[p].x += b4.x; x[p].y += b4.y; x[p].z += b4.z; x[p].w += b4.w; }
          }
          if (!B2B && !kNorm && P.gate) {
#pragma unroll
            for (int p = 0; p < 4; ++p) { x[p].x *= g4[p].x; x[p].y *= g4[p].y; x[p].z *= g4[p].z; x[p].w *= g4[p].w; }
          }
          if (kNorm && P.gate) {                // norm-producer instantiation: gate rows fetched at their use (L1/L2 hits)
            const float* g0 = P.gate + n;
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              const float4 g = __ldg(reinterpret_cast<const float4*>(g0 + item_p[p] * P.gate_ld));
              x[p].x *= g.x; x[p].y *= g.y; x[p].z *= g.z; x[p].w *= g.w;
            }
          }
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            x[p].x = fmaf(x[p].x, P.alpha, rr[p].x); x[p].y = fmaf(x[p].y, P.alpha, rr[p].y);
            x[p].z = fmaf(x[p].z, P.alpha, rr[p].z); x[p].w = fmaf(x[p].w, P.alpha, rr[p].w);
          }
          if (P.relu) {
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              x[p].x = fmaxf(x[p].x, 0.f); x[p].y = fmaxf(x[p].y, 0.f); x[p].z = fmaxf(x[p].z, 0.f); x[p].w = fmaxf(x[p].w, 0.f);
            }
          }
          if (P.out_f32) {
            float* o0 = P.out_f32 + row0 * P.out_f32_ld + n;
            const long long st = 4 * P.out_f32_ld;
#pragma unroll
            for (int p = 0; p < 4; ++p)
              if (4 * p < rl) *reinterpret_cast<float4*>(o0 + p * st) = x[p];
          }
          if (P.out_bf16) {
            __nv_bfloat16* o0 = P.out_bf16 + row0 * P.out_bf16_ld + n;
            const long long st = 4 * P.out_bf16_ld;
#pragma unroll
            for (int p = 0; p < 4; ++p)
              if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
          }
          if (kNorm && P.out_scaled) {   // the next GEMM's A operand: h * w_norm * (1 + scale); and sum h^2
            __nv_bfloat16* o0 = P.out_scaled + row0 * P.out_scaled_ld + n;
            const long long st = 4 * P.out_scaled_ld;
            const float* c0 = P.colscale + n;
            float (&sq)[4] = ssq[(c / 32) & 1];
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              const float4 c4 = __ldg(reinterpret_cast<const float4*>(c0 + item_p[p] * P.colscale_ld));
              sq[p] = fmaf(x[p].x, x[p].x, fmaf(x[p].y, x[p].y, fmaf(x[p].z, x[p].z, fmaf(x[p].w, x[p].w, sq[p]))));
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
            for (int p = 0; p < 4; ++p) {
              float s;
              s = __sinf(a4.x * x[p].x); x[p].x = fmaf(s * s, i4.x, x[p].x);
              s = __sinf(a4.y * x[p].y); x[p].y = fmaf(s * s, i4.y, x[p].y);
              s = __sinf(a4.z * x[p].z); x[p].z = fmaf(s * s, i4.z, x[p].z);
              s = __sinf(a4.w * x[p].w); x[p].w = fmaf(s * s, i4.w, x[p].w);
            }
#pragma unroll
            for (int p = 0; p < 4; ++p)
              if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
          }
#pragma unroll
          for (int p = 0; p < 4; ++p) rr[p] = rr_n[p];
        }
        if (kNorm && P.ssq_out) {   // the 8 lanes of a row hold 4 columns each: one partial per (row, n-tile, chunk parity)
#pragma unroll
          for (int par = 0; par < 2; ++par) {
#pragma unroll
            for (int p = 0; p < 4; ++p) {
              float sv = ssq[par][p];
              sv += __shfl_xor_sync(0xffffffffu, sv, 1);
              sv += __shfl_xor_sync(0xffffffffu, sv, 2);
              sv += __shfl_xor_sync(0xffffffffu, sv, 4);
              if ((lane & 7) == 0 && 4 * p < rl) P.ssq_out[(row0 + 4 * p) * P.ssq_ld + nt * 2 + par] = sv;
            }
          }
        }
      } else if constexpr (MODE == EPI_SWIGLU) {
        // tile columns: [32 gate | 32 up] pairs -> BN/2 outputs at column n0/2.  Gate column c + j and up column
        // c + 32 + j are fragment groups i and i + 4 of the same thread.
        float nrm_rstd[2] = {1.f, 1.f};   // fused RMSNorm of the fragment rows fr and fr + 8
        const float* nrm_brow[2] = {nullptr, nullptr};
        if (P.ssq_in) {
          nrm_row(fr, nrm_rstd[0], nrm_brow[0]);
          nrm_row(fr + 8, nrm_rstd[1], nrm_brow[1]);
        }
#pragma unroll
        for (int c = 0; c < BN; c += 64) {
          if (n0 + c >= P.N) break;
          float* g = &accr[c / 2];
          float* u = &accr[c / 2 + 16];
          if (P.ssq_in) {   // fused RMSNorm: rstd * acc + (shift @ W^T) of this row's item (L1-broadcast loads)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float2 bg = __ldg(reinterpret_cast<const float2*>(nrm_brow[h] + c + 8 * i + fc));
                const float2 bu = __ldg(reinterpret_cast<const float2*>(nrm_brow[h] + c + 32 + 8 * i + fc));
                float* gi = g + 4 * i + 2 * h;
                float* ui = u + 4 * i + 2 * h;
                gi[0] = fmaf(gi[0], nrm_rstd[h], bg.x); gi[1] = fmaf(gi[1], nrm_rstd[h], bg.y);
                ui[0] = fmaf(ui[0], nrm_rstd[h], bu.x); ui[1] = fmaf(ui[1], nrm_rstd[h], bu.y);
              }
            }
          }
#pragma unroll
          for (int j = 0; j < 16; ++j) g[j] = silu_f(g[j]) * u[j];
          float4 x[4];
          frag_put(g);
          stage_get(x);
          __nv_bfloat16* o0 = P.out_bf16 + row0 * P.out_bf16_ld + ((n0 + c) >> 1) + tr_c;
          const long long st = 4 * P.out_bf16_ld;
#pragma unroll
          for (int p = 0; p < 4; ++p)
            if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
        }
      } else {  // EPI_QKV: each 128-col group is one head; a thread holds 32 of its columns for two rows
        int pos[4];                             // RoPE position of each pass (one modulo per tile)
#pragma unroll
        for (int p = 0; p < 4; ++p) pos[p] = (int)(((uint32_t)row0 + 4u * p) % (uint32_t)P.rope_T);   // rows < 2^31: no 64-bit division
        // Row form, for the per-row reductions: lane l reads row rr = l % 16 of a staged chunk (the two half-warps
        // mirror each other), so that every sum runs as one sequential chain over the row's columns, in column order.
        const int rr = lane & 15;
        auto row_get = [&](float (&v)[32]) {
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float4 t = lds128(epi_addr(rr, 4 * k));
            v[4 * k] = t.x; v[4 * k + 1] = t.y; v[4 * k + 2] = t.z; v[4 * k + 3] = t.w;
          }
        };
        float nrm_rstd = 1.f;     // fused RMSNorm of row rr
        const float* nrm_brow = nullptr;
        float nrs[4];             // ... and of each pass's row, with its item's bias row
        int nboff[4];
        if (P.ssq_in) {
          nrm_row(rr, nrm_rstd, nrm_brow);
#pragma unroll
          for (int p = 0; p < 4; ++p) {
            nrs[p] = __shfl_sync(0xffffffffu, nrm_rstd, 4 * p + tr_r);
            nboff[p] = (4 * p < rl) ? (int)((uint32_t)(row0 + 4 * p) / (uint32_t)P.ibias_div) * (int)P.ibias_ld : 0;
          }
        }
#pragma unroll
        for (int hc = 0; hc < BN; hc += 128) {
          const int nh = n0 + hc;
          if (nh >= P.N) break;
          float* acc_h = &accr[hc / 2];   // the head's 64 fragment values: group i (cols 8i + fc, +1) at acc_h[4i ..]
          const int rep = P.qkv_period > 0 ? nh / P.qkv_period : 0;
          const int nhp = P.qkv_period > 0 ? nh - rep * P.qkv_period : nh;
          const float* nw = (nhp < P.n_q_end) ? P.qnorm_w + rep * P.norm_w_stride
                                               : (nhp < P.n_k_end ? P.knorm_w + rep * P.norm_w_stride : nullptr);
          if (XAP || P.xa_kv != nullptr) {
            // ---- fused cross-attention to the row's text tokens (scores are linear in the un-normalised query).
            //      Scores in row form: both half-warps run the row's sum of squares, each the dot products of
            //      half of the tokens (j0 .. j0+3) ----
            const int b_r = (int)((uint32_t)row_grow(rr) / (uint32_t)P.xa_T);
            const __nv_bfloat16* kp_r = P.xa_kv + (long long)b_r * P.xa_Tk * P.xa_kv_ld + nh;
            const int j0 = (lane >> 4) * (XA_MAX_TK / 2);
            float ss = 0.f, sh[XA_MAX_TK / 2];
#pragma unroll
            for (int jj = 0; jj < XA_MAX_TK / 2; ++jj) sh[jj] = 0.f;
#pragma unroll
            for (int c = 0; c < 128; c += 32) {
              frag_put(acc_h + c / 2);
              float v[32];
              row_get(v);
#pragma unroll
              for (int i = 0; i < 32; i += 4) {
                const float4 w4 = __ldg(reinterpret_cast<const float4*>(nw + c + i));
                ss = fmaf(v[i], v[i], ss); ss = fmaf(v[i + 1], v[i + 1], ss);
                ss = fmaf(v[i + 2], v[i + 2], ss); ss = fmaf(v[i + 3], v[i + 3], ss);
                v[i] *= w4.x; v[i + 1] *= w4.y; v[i + 2] *= w4.z; v[i + 3] *= w4.w;
              }
#pragma unroll
              for (int jj = 0; jj < XA_MAX_TK / 2; ++jj) {
                if (j0 + jj < P.xa_Tk) {
                  const uint4* kr = reinterpret_cast<const uint4*>(kp_r + (long long)(j0 + jj) * P.xa_kv_ld + c);
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
                  sh[jj] += d;
                }
              }
            }
            float sc[XA_MAX_TK];   // all tokens of row rr: this half-warp's and, from lane ^ 16, the other's
#pragma unroll
            for (int jj = 0; jj < XA_MAX_TK / 2; ++jj) {
              const float o = __shfl_xor_sync(0xffffffffu, sh[jj], 16);
              sc[jj] = j0 == 0 ? sh[jj] : o;
              sc[XA_MAX_TK / 2 + jj] = j0 == 0 ? o : sh[jj];
            }
            const float rstd = rsqrtf(ss * (1.f / 128.f) + P.eps);
            float mx = -INFINITY;
#pragma unroll
            for (int j = 0; j < XA_MAX_TK; ++j) {
              const bool ok = j < P.xa_Tk && (!P.xa_mask || P.xa_mask[(long long)b_r * P.xa_Tk + j]);
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
            if constexpr (XAP) {   // probabilities only: lanes 0..15 hold rows 0..15 of the warp, Tk values each
              if (lane < 16 && t_base + rr < P.rows_per_item) {
                __nv_bfloat16* pp = P.xa_p + row_grow(rr) * P.xa_p_ld + (nh >> 7);
#pragma unroll
                for (int j = 0; j < XA_MAX_TK; ++j)
                  if (j < P.xa_Tk) pp[j * (P.N >> 7)] = __float2bfloat16_rn(sc[j] * inv);
              }
            } else {
            // O = P V in fragment form, accumulated over the head's (no longer needed) accumulators: the
            // probabilities of the fragment rows fr and fr + 8 come from lanes fr and fr + 8
            float pf[2][XA_MAX_TK];
#pragma unroll
            for (int j = 0; j < XA_MAX_TK; ++j) {
              const float pj = sc[j] * inv;
              pf[0][j] = __shfl_sync(0xffffffffu, pj, fr);
              pf[1][j] = __shfl_sync(0xffffffffu, pj, fr + 8);
            }
#pragma unroll
            for (int i = 0; i < 64; ++i) acc_h[i] = 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int b = (int)((uint32_t)row_grow(fr + 8 * h) / (uint32_t)P.xa_T);
              const __nv_bfloat16* vp = P.xa_kv + (long long)b * P.xa_Tk * P.xa_kv_ld + nh + P.xa_v_col0 + fc;
#pragma unroll
              for (int j = 0; j < XA_MAX_TK; ++j) {
                if (j < P.xa_Tk) {
                  const __nv_bfloat16* vr = vp + (long long)j * P.xa_kv_ld;
#pragma unroll
                  for (int i = 0; i < 16; ++i) {
                    const uint32_t v2u = __ldg(reinterpret_cast<const unsigned int*>(vr + 8 * i));
                    const float2 v2 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v2u));
                    float& o0 = acc_h[4 * i + 2 * h];
                    float& o1 = acc_h[4 * i + 2 * h + 1];
                    o0 = fmaf(pf[h][j], v2.x, o0); o1 = fmaf(pf[h][j], v2.y, o1);
                  }
                }
              }
            }
#pragma unroll
            for (int c = 0; c < 128; c += 32) {
              float4 x[4];
              frag_put(acc_h + c / 2);
              stage_get(x);
              __nv_bfloat16* o0 = P.out_bf16 + row0 * P.out_bf16_ld + nh + c + tr_c;
              const long long st = 4 * P.out_bf16_ld;
#pragma unroll
              for (int p = 0; p < 4; ++p)
                if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
            }
            }
            continue;
          }
          if constexpr (XAP) continue;   // (never reached: XAP launches always carry xa_kv)
          float rs[4] = {1.f, 1.f, 1.f, 1.f};   // per-head RMSNorm rstd of each pass's row
          if (nw) {
            float ss = 0.f;   // of row rr, over the head's 128 columns in order
#pragma unroll
            for (int c = 0; c < 128; c += 32) {
              frag_put(acc_h + c / 2);
              float v[32];
              row_get(v);
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
            const float rstd = rsqrtf(ss * (1.f / 128.f) + P.eps);
#pragma unroll
            for (int p = 0; p < 4; ++p) rs[p] = __shfl_sync(0xffffffffu, rstd, 4 * p + tr_r);
          }
#pragma unroll
          for (int c = 0; c < 128; c += 32) {
            const int cc = c + tr_c;              // column inside the head
            float4 x[4];
            frag_put(acc_h + c / 2);
            stage_get(x);
            if (P.ssq_in) {
              const float* b0 = P.ibias + nh + cc;
#pragma unroll
              for (int p = 0; p < 4; ++p) {
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(b0 + nboff[p]));
                x[p].x = fmaf(x[p].x, nrs[p], b4.x); x[p].y = fmaf(x[p].y, nrs[p], b4.y);
                x[p].z = fmaf(x[p].z, nrs[p], b4.z); x[p].w = fmaf(x[p].w, nrs[p], b4.w);
              }
            }
            if (nw) {
              const float4 w4 = __ldg(reinterpret_cast<const float4*>(nw + cc));
#pragma unroll
              for (int p = 0; p < 4; ++p) {
                x[p].x *= rs[p] * w4.x; x[p].y *= rs[p] * w4.y; x[p].z *= rs[p] * w4.z; x[p].w *= rs[p] * w4.w;
              }
              if (P.use_rope) {
#pragma unroll
                for (int p = 0; p < 4; ++p) {
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
            for (int p = 0; p < 4; ++p)
              if (4 * p < rl) *reinterpret_cast<uint2*>(o0 + p * st) = pack4_bf16(x[p]);
          }
        }
      }
    }
  }

  if constexpr (CG == 2) cluster_sync_all(); else __syncthreads();
}

}  // namespace sab
