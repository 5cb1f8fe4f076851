// Cross-attention output projection folded into the text values (once per evaluation, all layers in one launch):
//
//     Ut[l][b*d + n][j*H + h] = bf16( sum_c Wo_l[n, h*128 + c] * V_l[b*L + j, h*128 + c] )
//
// Each head's attention output is a convex combination of the clip's L <= 8 value rows, so
//     cross.wo(O)[row, n] = sum_{h,j} p[row, h, j] * Ut[clip(row)][n, j*H + h]
// and the d x d output projection becomes a GEMM with K = H*L against a per-clip B operand (gemm_tc.cuh b_clip_rows).
// The columns are token-major (j*H + h, as the probabilities the cross.wq epilogue writes): a token's column does not
// depend on L, so a clip gets the same products in the same k positions whatever text length its batch is padded to,
// and its result does not depend on the batch.
//
// mma.sync m16n8k16 (bf16 in, fp32 accumulate): A = 16 rows of Wo x 16 columns of one head, B = the 16 x 8 block of
// V^T of one clip (token j is MMA column j; columns >= L are zero).  A CTA owns 32 output rows n of one layer; its 8
// warps take the heads round-robin and keep a head's A fragments (32 rows x 128 columns, 64 registers) while they sweep
// a chunk of clips.  Results go to a shared-memory copy of the chunk's Ut rows (32 rows x ldu per clip), which is
// written back with 16-byte stores once every head is in, so each Ut row leaves the SM whole.
#pragma once
#include "common.cuh"
#include "attention.cuh"   // mma_bf16_16816

namespace sab {

constexpr int XF_ROWS = 32;       // output rows n per CTA
constexpr int XF_THREADS = 256;   // 8 warps

struct XaFoldParams {
  const __nv_bfloat16* const* wo;   // [layers] -> packed cross_attention.wo [d, d] (K columns head-major)
  const __nv_bfloat16* kv;          // V of layer l: kv[(b*L + j) * kv_ld + l * kv_layer_cols + v_col0 + c]
  long long kv_ld, kv_layer_cols;
  int v_col0;
  __nv_bfloat16* ut;                // Ut of layer l: ut + l * ut_layer_stride, rows b*d + n, pitch ldu, column j*heads + h
  long long ut_layer_stride;
  int ldu;                          // >= heads * L, multiple of 8; columns [heads * L, ldu) are written as 0
  int d, heads, L, clips;
  int chunk;                        // clips per shared-memory chunk
};

SAB_DEVICE uint32_t ldg_u32(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); }

// grid (d / XF_ROWS, layers), XF_THREADS threads, chunk * XF_ROWS * ldu * 2 bytes of dynamic shared memory
__global__ void __launch_bounds__(XF_THREADS, 2) xattn_fold_kernel(const XaFoldParams P) {
  extern __shared__ __align__(16) __nv_bfloat16 xf_stage[];   // [chunk][XF_ROWS][ldu]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;          // fragment row / column-pair index
  const int n0 = blockIdx.x * XF_ROWS, l = blockIdx.y;
  const int ldu = P.ldu, L = P.L, H = P.heads;
  const __nv_bfloat16* wo = P.wo[l];
  const __nv_bfloat16* vbase = P.kv + l * P.kv_layer_cols + P.v_col0;
  __nv_bfloat16* ut = P.ut + l * P.ut_layer_stride;
  const int stage_elems = P.chunk * XF_ROWS * ldu;

  // the padding columns stay zero (no MMA result lands there)
  for (int i = threadIdx.x * 8; i < stage_elems; i += XF_THREADS * 8)
    *reinterpret_cast<uint4*>(xf_stage + i) = make_uint4(0u, 0u, 0u, 0u);
  __syncthreads();

  for (int c0 = 0; c0 < P.clips; c0 += P.chunk) {
    const int nb = min(P.chunk, P.clips - c0);
    for (int h = warp; h < P.heads; h += XF_THREADS / 32) {
      // A fragments of the 32 x 128 block Wo[n0 .., h*128 ..]: [m-tile][k-step][4]
      uint32_t a[2][8][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const __nv_bfloat16* w0 = wo + (long long)(n0 + mt * 16 + g) * P.d + h * 128 + 2 * t;
        const __nv_bfloat16* w8 = w0 + 8LL * P.d;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
          a[mt][ks][0] = ldg_u32(w0 + ks * 16);
          a[mt][ks][1] = ldg_u32(w8 + ks * 16);
          a[mt][ks][2] = ldg_u32(w0 + ks * 16 + 8);
          a[mt][ks][3] = ldg_u32(w8 + ks * 16 + 8);
        }
      }
      for (int bl = 0; bl < nb; ++bl) {
        // B fragments: token g of the clip (zero for g >= L), columns 2t, 2t+1 (+8) of each 16-wide k-step
        uint32_t bf[8][2];
        const bool tok = g < L;
        const __nv_bfloat16* vr = vbase + (long long)((c0 + bl) * L + (tok ? g : 0)) * P.kv_ld + h * 128 + 2 * t;
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
          bf[ks][0] = tok ? ldg_u32(vr + ks * 16) : 0u;
          bf[ks][1] = tok ? ldg_u32(vr + ks * 16 + 8) : 0u;
        }
        __nv_bfloat16* srow = xf_stage + (bl * XF_ROWS) * ldu + h;
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int ks = 0; ks < 8; ++ks) mma_bf16_16816(acc, a[mt][ks], bf[ks][0], bf[ks][1]);
          // acc: (row g, tokens 2t, 2t+1), (row g + 8, same tokens)
          const int r = mt * 16 + g, j = 2 * t;
          if (j < L) {
            srow[r * ldu + j * H] = __float2bfloat16_rn(acc[0]);
            srow[(r + 8) * ldu + j * H] = __float2bfloat16_rn(acc[2]);
          }
          if (j + 1 < L) {
            srow[r * ldu + (j + 1) * H] = __float2bfloat16_rn(acc[1]);
            srow[(r + 8) * ldu + (j + 1) * H] = __float2bfloat16_rn(acc[3]);
          }
        }
      }
    }
    __syncthreads();
    // clip b's 32 rows are one contiguous run of Ut: rows b*d + n0 .. n0+31
    const int run = XF_ROWS * ldu;   // elements, a multiple of 256
    for (int bl = 0; bl < nb; ++bl) {
      const uint4* src = reinterpret_cast<const uint4*>(xf_stage + bl * run);
      uint4* dst = reinterpret_cast<uint4*>(ut + ((long long)(c0 + bl) * P.d + n0) * ldu);
      for (int i = threadIdx.x; i < run / 8; i += XF_THREADS) dst[i] = src[i];
    }
    __syncthreads();
  }
}

}  // namespace sab
