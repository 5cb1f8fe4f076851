// libsamaudio_b200.so — engine + C ABI (include/samaudio_b200.h).
// Weights are repacked to bf16 GEMM operands at load; every (Bc, T, L) shape gets a static plan
// (workspace + TMA descriptors + launch records) that each ODE evaluation replays.
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <functional>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <array>

#include "../../include/samaudio_b200.h"
#include "host_util.h"
#include "attention.cuh"
#include "attention_tc2.cuh"
#include "attention_stream_tc.cuh"
#include "elementwise.cuh"
#include "codec_kernels.cuh"
#include "vision_kernels.cuh"
#include "xattn_fold.cuh"
#include "blend_windows.cuh"
#include "resample.cuh"
#include "spread_channels.cuh"

using namespace sab;
typedef __nv_bfloat16 bf16;

static thread_local std::string g_last_error;

// ---- per-device state (several engines on different GPUs may live in one process) ----
constexpr int kMaxDevices = 64;
static int cur_device() {
  int d = 0;
  SAB_CUDA(cudaGetDevice(&d));
  SAB_CHECK(d >= 0 && d < kMaxDevices, "device index %d out of range", d);
  return d;
}
static int sm_count() {   // of the current device
  static int cached[kMaxDevices] = {0};
  const int d = cur_device();
  if (!cached[d]) {
    cudaDeviceProp prop;
    SAB_CUDA(cudaGetDeviceProperties(&prop, d));
    cached[d] = prop.multiProcessorCount;
  }
  return cached[d];
}
// cudaFuncSetAttribute is per device: once per (kernel, device).  Keyed by the function ADDRESS: all instantiations
// of one kernel template share a function-pointer type, so a per-type static would configure only the first one.
static void ensure_dynamic_smem(const void* kern, int smem) {
  static std::unordered_map<const void*, std::array<bool, kMaxDevices>> configured;
  const int d = cur_device();
  auto& flags = configured[kern];   // value-initialised to all false on first use
  if (!flags[d]) {
    SAB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    flags[d] = true;
  }
}
// every entry point runs on its engine's device whatever the caller's current device is, and restores it
struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    int cur = 0;
    SAB_CUDA(cudaGetDevice(&cur));
    if (cur != dev) { SAB_CUDA(cudaSetDevice(dev)); prev = cur; }
  }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

// =====================================================================================================
// GEMM dispatch
// =====================================================================================================
template <int BN, int BK, int MODE, int CG, bool B2B = false, bool XAP = false>
static void launch_gemm_inst(const GemmOp& op, cudaStream_t st) {
  auto kern = gemm_tc_kernel<BN, BK, MODE, CG, B2B, XAP>;
  constexpr int smem = GemmSmem<BN, BK, CG, B2B>::kTotal;
  ensure_dynamic_smem(reinterpret_cast<const void*>(kern), smem);
  if (CG == 1) {
    kern<<<op.grid, GEMM_THREADS, smem, st>>>(op.tmA, op.tmB, op.b2b ? op.tmW : op.tmB, op.P);
  } else {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(op.grid);
    cfg.blockDim = dim3(GEMM_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = CG;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    SAB_CUDA(cudaLaunchKernelEx(&cfg, kern, op.tmA, op.tmB, op.tmB, op.P));
  }
  SAB_CUDA(cudaGetLastError());
}

// the instantiation table: the launcher of (BN, BK, mode, cg, b2b, xap = cross-attention probabilities out), or nullptr
// if that combination is not built
typedef void (*GemmLauncher)(const GemmOp&, cudaStream_t);
static GemmLauncher gemm_launcher(int BN, int BK, int mode, int cg, bool b2b, bool xap) {
  if (xap) {
    if (BN != 256 || BK != 64 || mode != EPI_QKV || b2b) return nullptr;
    if (cg == 2) return launch_gemm_inst<256, 64, EPI_QKV, 2, false, true>;
    if (cg == 1) return launch_gemm_inst<256, 64, EPI_QKV, 1, false, true>;
    return nullptr;
  }
  if (b2b) {
    if (mode != EPI_AFFINE || cg != 1) return nullptr;
    if (BN == 64 && BK == 64) return launch_gemm_inst<64, 64, EPI_AFFINE, 1, true>;
    if (BN == 96 && BK == 32) return launch_gemm_inst<96, 32, EPI_AFFINE, 1, true>;
    if (BN == 128 && BK == 64) return launch_gemm_inst<128, 64, EPI_AFFINE, 1, true>;
    return nullptr;
  }
#define SAB_CASE(bn_, bk_, md_, cg_) \
  if (BN == bn_ && BK == bk_ && mode == md_ && cg == cg_) return launch_gemm_inst<bn_, bk_, md_, cg_>;
  SAB_CASE(256, 64, EPI_AFFINE, 2)
  SAB_CASE(256, 64, EPI_AFFINE_NORM, 2)
  SAB_CASE(256, 64, EPI_AFFINE_NORM, 1)
  SAB_CASE(256, 64, EPI_SWIGLU, 2)
  SAB_CASE(256, 64, EPI_QKV, 2)
  SAB_CASE(256, 64, EPI_AFFINE, 1)
  SAB_CASE(192, 64, EPI_AFFINE, 1)
  SAB_CASE(128, 64, EPI_AFFINE, 1)
  SAB_CASE(96, 64, EPI_AFFINE, 1)
  SAB_CASE(64, 64, EPI_AFFINE, 1)
  SAB_CASE(96, 32, EPI_AFFINE, 1)
  SAB_CASE(128, 32, EPI_AFFINE, 1)
  SAB_CASE(256, 64, EPI_SWIGLU, 1)
  SAB_CASE(256, 64, EPI_QKV, 1)
  SAB_CASE(128, 64, EPI_QKV, 1)
#undef SAB_CASE
  return nullptr;
}

// Parameter combinations that the kernel would ignore, or turn into wrong results or stray reads, without an error
// (beyond what the instantiations' static_asserts cover).  Every launch is checked; host-only (no CUDA call), so the
// test seam can check a descriptor before it touches the device.
static void check_gemm(const char* tag, int BN, int BK, int mode, int cg, bool b2b, int grid, const GemmParams& P) {
  const bool affine = (mode == EPI_AFFINE || mode == EPI_AFFINE_NORM);
  SAB_CHECK(mode >= EPI_AFFINE && mode <= EPI_AFFINE_NORM, "%s: unknown GEMM mode %d", tag, mode);
  SAB_CHECK(P.N > 0 && P.N % 32 == 0, "%s: N=%d must be a positive multiple of 32", tag, P.N);
  SAB_CHECK(mode != EPI_QKV || P.N % 128 == 0, "%s: QKV mode needs whole 128-column heads (N=%d)", tag, P.N);
  SAB_CHECK(mode != EPI_SWIGLU || P.N % 64 == 0, "%s: SwiGLU mode needs whole [32 gate | 32 up] pairs (N=%d)", tag, P.N);
  SAB_CHECK(!P.xa_p || P.xa_kv, "%s: xa_p (cross-attention probabilities) needs fused cross-attention (xa_kv)", tag);
  SAB_CHECK(affine || P.out_bf16 || P.xa_p, "%s: SwiGLU / QKV modes write out_bf16, which is not set", tag);
  SAB_CHECK(P.b_clip_rows >= 0, "%s: b_clip_rows=%d must be >= 0", tag, P.b_clip_rows);
  if (P.b_clip_rows > 0) {
    SAB_CHECK(P.b_clip_div >= 1, "%s: b_clip_div=%d must be >= 1 with a per-clip B (b_clip_rows=%d)", tag, P.b_clip_div,
              P.b_clip_rows);
    SAB_CHECK(P.b_clip_rows >= P.N, "%s: b_clip_rows=%d must be >= N=%d (a clip's B holds all N rows)", tag,
              P.b_clip_rows, P.N);
    SAB_CHECK(!b2b, "%s: back-to-back tiles have no per-clip B", tag);
  }
  SAB_CHECK(!P.out_act || P.snake_alpha, "%s: out_act needs snake_alpha", tag);
  SAB_CHECK(mode == EPI_AFFINE_NORM || (!P.out_scaled && !P.ssq_out),
            "%s: the fused-norm producer outputs (out_scaled, ssq_out) need the AFFINE_NORM mode", tag);
  SAB_CHECK(!P.out_scaled || P.colscale, "%s: out_scaled needs colscale", tag);
  SAB_CHECK(!(P.gate || P.out_scaled) || P.gate_div > 0, "%s: gate_div=%d must be > 0", tag, P.gate_div);
  // the fused-norm consumer (rstd * acc + ibias) exists in the SwiGLU and plain QKV epilogues only
  SAB_CHECK(!(P.ssq_in && affine), "%s: the fused-norm consumer (ssq_in) is not applied in the affine modes", tag);
  SAB_CHECK(!(P.ssq_in && P.xa_kv), "%s: the fused-norm consumer (ssq_in) is not applied with fused cross-attention (xa_kv)", tag);
  SAB_CHECK(!P.ssq_in || (P.ssq_n > 0 && P.ibias), "%s: ssq_in needs ssq_n > 0 and ibias", tag);
  SAB_CHECK(!P.ibias || P.ibias_div > 0, "%s: ibias_div=%d must be > 0", tag, P.ibias_div);
  if (mode == EPI_QKV) {
    SAB_CHECK(!P.use_rope || (P.rope && P.rope_T > 0), "%s: use_rope needs rope and rope_T > 0", tag);
    SAB_CHECK(P.rope_T > 0, "%s: rope_T=%d must be > 0 (RoPE positions are row %% rope_T)", tag, P.rope_T);
  }
  if (P.xa_kv) {
    SAB_CHECK(mode == EPI_QKV, "%s: fused cross-attention (xa_kv) needs the QKV mode", tag);
    SAB_CHECK(P.xa_Tk >= 1 && P.xa_Tk <= XA_MAX_TK, "%s: xa_Tk=%d outside 1..%d", tag, P.xa_Tk, XA_MAX_TK);
    SAB_CHECK(P.xa_T >= 1, "%s: xa_T=%d must be >= 1", tag, P.xa_T);
    SAB_CHECK(P.qnorm_w && P.n_q_end >= P.N, "%s: fused cross-attention needs q-norm weights on every column", tag);
    SAB_CHECK(!P.xa_p || P.xa_p_ld >= (long long)(P.N / 128) * P.xa_Tk,
              "%s: xa_p_ld=%lld is below heads * xa_Tk = %d", tag, P.xa_p_ld, (P.N / 128) * P.xa_Tk);
  }
  if (b2b) {
    SAB_CHECK(BN == P.N, "%s: back-to-back tiles need BN == N (BN=%d, N=%d)", tag, BN, P.N);
    SAB_CHECK(cg == 1, "%s: back-to-back tiles need cg == 1 (cg=%d)", tag, cg);
    SAB_CHECK(mode == EPI_AFFINE, "%s: back-to-back tiles need the affine mode (mode=%d)", tag, mode);
    SAB_CHECK(!P.gate, "%s: back-to-back tiles apply no gate", tag);
    SAB_CHECK(P.b2b_bias && P.b2b_alpha, "%s: back-to-back tiles need b2b_bias and b2b_alpha", tag);
  }
  SAB_CHECK(cg == 1 || cg == 2, "%s: cg=%d must be 1 or 2", tag, cg);
  SAB_CHECK(grid > 0 && grid % cg == 0, "%s: grid of %d CTAs is not a multiple of cg=%d", tag, grid, cg);
  SAB_CHECK(P.group_m >= 1 && (P.reverse_m == 0 || P.reverse_m == 1), "%s: group_m=%d / reverse_m=%d out of range", tag,
            P.group_m, P.reverse_m);
  int kb[2] = {0, 0};
  for (int l = 0; l < 2; ++l) {
    SAB_CHECK(P.n_runs[l] >= 0 && P.n_runs[l] <= GEMM_MAX_RUNS, "%s: %d K runs (at most %d)", tag, P.n_runs[l],
              GEMM_MAX_RUNS);
    for (int r = 0; r < P.n_runs[l]; ++r) {
      SAB_CHECK(P.runs[l][r].nkb > 0, "%s: K run with %d k-blocks", tag, P.runs[l][r].nkb);
      kb[l] += P.runs[l][r].nkb;
    }
  }
  SAB_CHECK(kb[0] > 0, "%s: empty K run list", tag);
  if (P.n_period > 0) {
    SAB_CHECK(kb[1] == kb[0], "%s: run lists differ in K (%d vs %d k-blocks)", tag, kb[0], kb[1]);
    SAB_CHECK(P.n_switch % BN == 0 && P.n_period % BN == 0, "%s: BN=%d does not divide the tap switch %d/%d", tag, BN,
              P.n_switch, P.n_period);
  }
  SAB_CHECK(gemm_launcher(BN, BK, mode, cg, b2b, P.xa_p != nullptr) != nullptr,
            "%s: no GEMM instantiation for BN=%d BK=%d mode=%d cg=%d b2b=%d%s", tag, BN, BK, mode, cg, (int)b2b,
            P.xa_p ? " with xa_p" : "");
}

static void launch_gemm(const GemmOp& op, cudaStream_t st) {
  check_gemm(op.tag, op.BN, op.BK, op.mode, op.cg, op.b2b, op.grid, op.P);
  gemm_launcher(op.BN, op.BK, op.mode, op.cg, op.b2b, op.P.xa_p != nullptr)(op, st);
}

// A operand view
struct AView {
  const bf16* ptr;
  int64_t cols;        // row width visible to TMA (elements)
  int64_t rows;        // rows per item
  int64_t items;
  int64_t row_pitch;   // elements
  int64_t item_pitch;  // elements
};
static AView flat_view(const bf16* p, int64_t M, int64_t K, int64_t ld = -1) {
  return AView{p, K, M, 1, ld < 0 ? K : ld, 0};
}
static AView seq_view(const bf16* p, int64_t items, int64_t T, int64_t C) { return AView{p, C, T, items, C, T * C}; }

struct RunList {
  int n[2] = {0, 0};
  KRun r[2][GEMM_MAX_RUNS];
  int period = 0, sw = 0;
  void add(int list, int shift, int col, int nkb) {
    SAB_CHECK(n[list] < GEMM_MAX_RUNS, "too many K runs");
    r[list][n[list]++] = KRun{shift, col, nkb};
  }
  int total_kb(int list) const {
    int t = 0;
    for (int i = 0; i < n[list]; ++i) t += r[list][i].nkb;
    return t;
  }
};

static int g_force_cg = 0;   // SAB_FORCE_CG=1|2 overrides the automatic CTA-group choice (A/B measurements)

// cg = 0: the automatic choice — 2-CTA clusters (256 x BN tiles, B tile multicast to both CTAs) for the big
// tensor-bound GEMMs, unless SAB_FORCE_CG overrides it.  An explicit cg always wins.
static int pick_cg(const AView& A, int BN, int BK, int cg) {
  if (cg != 0) return cg;
  if (BN != 256 || BK != 64) return 1;
  if (g_force_cg) return g_force_cg;
  return (A.rows * A.items >= 1024 && A.rows >= 200) ? 2 : 1;
}

static GemmOp make_gemm(const char* tag, const AView& A, const bf16* B, int N, int BN, int BK, int mode,
                        const RunList& runs, int cg = 0) {
  GemmOp op;
  memset(&op.P, 0, sizeof(op.P));
  op.tag = tag;
  op.BN = BN; op.BK = BK; op.mode = mode;
  cg = pick_cg(A, BN, BK, cg);
  op.cg = cg;
  const int ktot = runs.total_kb(0) * BK;
  if (runs.period > 0) SAB_CHECK(runs.total_kb(1) * BK == ktot, "%s: run lists differ in K", tag);
  op.tmA = make_tmap_3d(A.ptr, A.cols, A.rows, A.items, A.row_pitch, A.item_pitch == 0 ? A.rows * A.row_pitch : A.item_pitch,
                        BK, GEMM_BM);
  op.tmB = make_tmap_2d(B, ktot, N, ktot, BK, BN / cg);
  GemmParams& P = op.P;
  P.rows_per_item = (int)A.rows;
  P.n_items = (int)A.items;
  P.tiles_per_item = (int)((A.rows + GEMM_BM * cg - 1) / (GEMM_BM * cg));
  P.N = N;
  P.n_tiles_n = (N + BN - 1) / BN;
  // rasterisation: keep one group's A panel (group_m x 128*cg x K bf16) around 24 MB so it stays L2-resident
  {
    const double panel_bytes = (double)GEMM_BM * cg * ktot * 2.0;
    int gm = (int)(24.0e6 / panel_bytes);
    gm = gm < 4 ? 4 : (gm > 32 ? 32 : gm);
    P.group_m = gm;
  }
  for (int l = 0; l < 2; ++l) {
    P.n_runs[l] = runs.n[l];
    for (int i = 0; i < runs.n[l]; ++i) P.runs[l][i] = runs.r[l][i];
  }
  P.n_period = runs.period;
  P.n_switch = runs.sw;
  if (runs.period > 0) SAB_CHECK(runs.sw % BN == 0 && runs.period % BN == 0, "%s: BN=%d does not divide the tap switch %d/%d", tag, BN, runs.sw, runs.period);
  P.alpha = 1.f;
  P.gate_div = 1;
  P.eps = 1e-5f;
  const long long tiles = (long long)P.n_items * P.tiles_per_item * P.n_tiles_n;
  op.grid = (int)std::min<long long>(tiles, sm_count() / cg) * cg;
  op.flops = 2.0 * (double)A.rows * (double)A.items * (double)N * (double)ktot;
  op.rows = (double)A.rows * (double)A.items;
  op.in_bytes = op.rows * (double)A.cols * 2.0 + (double)N * (double)ktot * 2.0;
  SAB_CHECK(N % 32 == 0, "%s: N=%d must be a multiple of 32", tag, N);
  return op;
}
static GemmOp make_linear(const char* tag, const bf16* A, int64_t M, int K, const bf16* B, int N, int BN, int mode,
                          int64_t lda = -1) {
  SAB_CHECK(K % 64 == 0, "%s: K=%d must be a multiple of 64", tag, K);
  RunList rl;
  rl.add(0, 0, 0, K / 64);
  return make_gemm(tag, flat_view(A, M, K, lda), B, N, BN, 64, mode, rl);
}
// Per-clip B: item i of the GEMM multiplies rows (i / clip_div) * clip_rows + [0, N) of B [n_clips * clip_rows, b_cols]
// (row pitch b_ld elements; TMA zero-fills the k-block columns past b_cols).  FLOPs count K = b_cols and the bytes
// count each clip's B once.
static void set_per_clip_b(GemmOp& op, const bf16* B, int64_t b_cols, int64_t b_ld, int clip_rows, int clip_div) {
  SAB_CHECK(clip_rows > 0 && clip_div > 0, "%s: per-clip B needs clip_rows > 0 and clip_div > 0", op.tag);
  int ktot = 0;
  for (int r = 0; r < op.P.n_runs[0]; ++r) ktot += op.P.runs[0][r].nkb * op.BK;
  const int64_t n_clips = (op.P.n_items + clip_div - 1) / clip_div;
  op.tmB = make_tmap_2d(B, b_cols, n_clips * clip_rows, b_ld, op.BK, op.BN / op.cg);
  op.P.b_clip_rows = clip_rows;
  op.P.b_clip_div = clip_div;
  op.in_bytes += (double)op.P.N * ((double)n_clips * (double)b_cols - (double)ktot) * 2.0;
  op.flops = 2.0 * op.rows * (double)op.P.N * (double)b_cols;
}

// =====================================================================================================
// weight packing kernels
// =====================================================================================================
enum RowMap { ROW_IDENT = 0, ROW_HEADS = 1, ROW_SWIGLU_A = 2, ROW_SWIGLU_B = 3 };

// dst[(row0 + map(r)) * ld + col0 + c] = bf16(src[r*rs + c*cs])
__global__ void pack_bf16_kernel(bf16* __restrict__ dst, long long ld, long long row0, long long col0,
                                 const float* __restrict__ src, long long R, long long C, long long rs, long long cs,
                                 int rowmap, int H) {
  const long long n = R * C;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / C, c = i % C;
    long long pr = r;
    if (rowmap == ROW_HEADS) { const long long dd = r / H, h = r % H; pr = h * (R / H) + dd; }
    else if (rowmap == ROW_SWIGLU_A) pr = (r >> 5) * 64 + (r & 31);
    else if (rowmap == ROW_SWIGLU_B) pr = (r >> 5) * 64 + 32 + (r & 31);
    dst[(row0 + pr) * ld + col0 + c] = __float2bfloat16(src[r * rs + c * cs]);
  }
}
static void pack(bf16* dst, long long ld, long long row0, long long col0, const float* src, long long R, long long C,
                 long long rs, long long cs, int rowmap, int H, cudaStream_t st) {
  const long long n = R * C;
  const int grid = (int)std::min<long long>((n + 255) / 256, 4096);
  pack_bf16_kernel<<<grid, 256, 0, st>>>(dst, ld, row0, col0, src, R, C, rs, cs, rowmap, H);
  SAB_CUDA(cudaGetLastError());
}

// =====================================================================================================
// engine state
// =====================================================================================================
struct Slot {
  std::vector<int64_t> shape;
  std::function<void(const float*, cudaStream_t)> load;
  bool loaded = false;
};

struct LayerW {
  bf16 *wqkv, *wo, *wq_c, *wkv_c, *wo_c, *w13, *w2;
  float *qn, *kn, *qn_c, *kn_c, *attn_norm, *ffn_norm;
  float* qn_scaled = nullptr;   // q_norm.weight * log2(e)/sqrt(hd): the QKV epilogue emits q in the softmax's log2 domain
  // self-attention logit bound (log2 domain) from the QK-norm weights: |q.k| / sqrt(hd) <= sqrt(hd) max|w_q| max|w_k|
  // (RMSNorm'd vectors have norm <= sqrt(hd) max|w|, RoPE preserves norms); < 0: unknown -> exact two-pass softmax
  float att_shift_log2 = -1.f;
};

struct ConvLayer {   // a multi-channel codec conv lowered to the GEMM
  bf16* w = nullptr;
  float* bias = nullptr;
  int cin = 0, cout = 0, k = 0, stride = 1, dil = 1;
  bool transposed = false;
};
struct ResUnitW {
  float* a0; ConvLayer c7; float* a1; ConvLayer c1;
};
struct EncBlockW { ResUnitW ru[3]; float* a_down; ConvLayer down; int cin, cout, stride; };
struct DecBlockW { float* a_up; ConvLayer up; ResUnitW ru[3]; int cin, cout, stride; };

struct DitPlan;
struct CodecPlan;
struct ResampleTableDev { DevicePool pool; int o = 1, n = 1, K = 1; float* w = nullptr; int* lo = nullptr; };
struct ProfRec { const char* tag; double flops; double bytes; };

struct sab_engine {
  sab_config cfg;
  int device = 0;
  DevicePool wpool;
  std::unordered_map<std::string, Slot> slots;
  float* staging = nullptr;
  int64_t staging_elems = 0;
  bool finalized = false;
  int64_t launches = 0;
  cudaStream_t capture_stream = nullptr;   // private stream for graph capture (the caller's may be the NULL stream)
  bool prof = false;
  std::vector<ProfRec> prof_recs;
  std::vector<cudaEvent_t> prof_events;

  // --- DiT weights ---
  std::vector<LayerW> layers;
  float* tables = nullptr;          // [L, 6, d]
  bf16* wkv_c_all = nullptr;        // [L, 2d, d]
  float* kn_c_all = nullptr;        // [L, 128]
  bf16 *wp_y, *wp_f, *wmem, *wvid;  // proj (noisy third / feature third), memory_proj, align conv
  float *proj_b, *mem_b, *vid_b, *vid_ln_w, *vid_ln_b, *vid_gate, *vid_const;
  float *anchor_embed, *anchor_proj, *anchor_gate, *anchor_table;
  bf16 *xe_w[2]; float *xe_b[2], *xe_gn_w[2], *xe_gn_b[2];
  bf16 *t_w13, *t_w2, *tb_w, *y_w13, *y_w2, *w_out;
  float *tb_b, *final_norm, *final_table;
  float* norm_w_all = nullptr;      // [2L, d]: attention_norm / ffn_norm weights of every layer, contiguous (finalize)
  float2* rope = nullptr;
  int rope_len = 0;

  // --- codec weights ---
  float *enc0_w, *enc0_b;                 // Conv1d(1, C0, 7)
  std::vector<EncBlockW> enc_blocks;
  float* enc_final_alpha; ConvLayer enc_final;   // Snake + Conv k3
  ConvLayer in_proj, out_proj;            // in_proj packed as [2*cz, latent] (mean rows duplicated)
  ConvLayer dec0;                         // Conv k7 latent -> decoder_dim
  std::vector<DecBlockW> dec_blocks;
  float* dec_final_alpha; float *dec_last_w, *dec_last_b;  // Snake + Conv1d(C,1,7) + tanh

  // resident DiT plans, one per (B, candidates, T, L), least recently used evicted beyond max_dit_plans; `dit` is the
  // one the last sab_prepare filled, which sab_solve / sab_dit_forward run
  std::vector<std::unique_ptr<DitPlan>> dit_plans;
  DitPlan* dit = nullptr;
  std::map<std::pair<int, long long>, std::unique_ptr<CodecPlan>> enc_plans, dec_plans;
  int64_t plan_clock = 0;
  size_t max_dit_plans = 1, max_codec_plans = 3;   // sab_set_plan_limits
  int64_t dit_plan_builds = 0, graph_captures = 0, codec_plan_builds = 0;   // sab_plan_stats

  // sab_resample: one table per rate pair, kept until sab_destroy, and the device copy of a call's segment list
  std::map<std::pair<int, int>, std::unique_ptr<ResampleTableDev>> rs_tables;
  DevicePool rs_desc_pool;
  ResampleSeg* rs_desc = nullptr;
  int64_t rs_desc_cap = 0;

  // sab_spread_channels: the twiddle and window table (built on first use, kept until sab_destroy) and the device copy
  // of a call's segment list
  DevicePool sp_table_pool, sp_desc_pool;
  float2* sp_table = nullptr;
  SpreadSeg* sp_desc = nullptr;
  int64_t sp_desc_cap = 0;

  ~sab_engine();
};

// Every kernel launch goes through mark(): it counts the launch and, when profiling is on, drops one event
// in front of it; the time between consecutive events is attributed to the launch that follows the first.
static void mark(sab_engine* e, cudaStream_t st, const char* tag, double flops = 0, double bytes = 0) {
  e->launches++;
  if (!e->prof) return;
  if (e->prof_recs.size() >= e->prof_events.size()) {
    cudaEvent_t ev;
    SAB_CUDA(cudaEventCreate(&ev));
    e->prof_events.push_back(ev);
  }
  SAB_CUDA(cudaEventRecord(e->prof_events[e->prof_recs.size()], st));
  e->prof_recs.push_back(ProfRec{tag, flops, bytes});
}

// =====================================================================================================
// weight registry
// =====================================================================================================
static void reg(sab_engine* e, const std::string& name, std::vector<int64_t> shape,
                std::function<void(const float*, cudaStream_t)> fn) {
  Slot s;
  s.shape = std::move(shape);
  s.load = std::move(fn);
  e->slots[name] = std::move(s);
}
static void reg_f32(sab_engine* e, const std::string& name, std::vector<int64_t> shape, float** dst) {
  int64_t n = 1;
  for (auto v : shape) n *= v;
  *dst = e->wpool.alloc<float>(n, true);
  float* d = *dst;
  reg(e, name, shape, [d, n](const float* src, cudaStream_t st) {
    SAB_CUDA(cudaMemcpyAsync(d, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  });
}
// plain [out, in] linear -> bf16 [out, in] (optionally a column window of the source)
static void reg_linear(sab_engine* e, const std::string& name, int out, int in, bf16** dst, int rowmap = ROW_IDENT,
                       int H = 1, bf16* into = nullptr, long long row0 = 0, long long ld = -1, int src_col0 = 0,
                       int src_cols = -1) {
  const int cols = src_cols < 0 ? in : src_cols;
  if (!into) { *dst = e->wpool.alloc<bf16>((int64_t)out * cols, true); into = *dst; }
  if (ld < 0) ld = cols;
  reg(e, name, {out, in}, [=](const float* src, cudaStream_t st) {
    pack(into, ld, row0, 0, src + src_col0, out, cols, in, 1, rowmap, H, st);
  });
}
// Conv1d weight [co, ci, k] -> bf16 [co, k*ci] (tap-major K)
static void reg_conv(sab_engine* e, const std::string& name, ConvLayer* L, int co, int ci, int k, int stride, int dil) {
  L->cin = ci; L->cout = co; L->k = k; L->stride = stride; L->dil = dil; L->transposed = false;
  L->w = e->wpool.alloc<bf16>((int64_t)co * ci * k, true);
  bf16* w = L->w;
  reg(e, name + ".weight", {co, ci, k}, [=](const float* src, cudaStream_t st) {
    for (int kk = 0; kk < k; ++kk) pack(w, (long long)k * ci, 0, (long long)kk * ci, src + kk, co, ci, (long long)ci * k, k, ROW_IDENT, 1, st);
  });
  reg_f32(e, name + ".bias", {co}, &L->bias);
}
// ConvTranspose1d weight [ci, co, 2s] (stride s, padding s/2) -> bf16 [s*co, 2*ci]:
// output sample r*s+u is x[r] * W[:, :, u+p] + (u < s/2 ? x[r-1] * W[:, :, u+p+s] : x[r+1] * W[:, :, u+p-s])
static void reg_convT(sab_engine* e, const std::string& name, ConvLayer* L, int ci, int co, int s) {
  SAB_CHECK(s % 2 == 0, "codec rates must be even (got %d)", s);
  L->cin = ci; L->cout = co; L->k = 2 * s; L->stride = s; L->dil = 1; L->transposed = true;
  L->w = e->wpool.alloc<bf16>((int64_t)s * co * 2 * ci, true);
  bf16* w = L->w;
  const int K = 2 * s, p = s / 2;
  reg(e, name + ".weight", {ci, co, K}, [=](const float* src, cudaStream_t st) {
    for (int u = 0; u < s; ++u) {
      const int k0 = u + p;
      const int k1 = (u < s / 2) ? u + p + s : u + p - s;
      pack(w, 2LL * ci, (long long)u * co, 0, src + k0, co, ci, K, (long long)co * K, ROW_IDENT, 1, st);
      pack(w, 2LL * ci, (long long)u * co, ci, src + k1, co, ci, K, (long long)co * K, ROW_IDENT, 1, st);
    }
  });
  reg_f32(e, name + ".bias", {co}, &L->bias);
}
static void reg_resunit(sab_engine* e, const std::string& p, ResUnitW* R, int c, int dil) {
  reg_f32(e, p + ".block.0.alpha", {1, c, 1}, &R->a0);
  reg_conv(e, p + ".block.1", &R->c7, c, c, 7, 1, dil);
  reg_f32(e, p + ".block.2.alpha", {1, c, 1}, &R->a1);
  reg_conv(e, p + ".block.3", &R->c1, c, c, 1, 1, 1);
}

static void register_weights(sab_engine* e) {
  const sab_config& c = e->cfg;
  const int d = c.dim, H = c.n_heads, hid = c.ffn_hidden, L = c.n_layers;
  auto S = [](const char* f, int i) { return fmt(f, i); };
  // ---- conditioning ----
  e->wp_y = e->wpool.alloc<bf16>((int64_t)d * 256, true);
  e->wp_f = e->wpool.alloc<bf16>((int64_t)d * 256, true);
  SAB_CHECK(c.in_channels == 768 && c.out_channels == 256, "in_channels/out_channels must be 768/256");
  {
    bf16 *wy = e->wp_y, *wf = e->wp_f;
    const int in = c.in_channels;
    reg(e, "proj.weight", {d, in}, [=](const float* src, cudaStream_t st) {
      pack(wy, 256, 0, 0, src, d, 256, in, 1, ROW_IDENT, 1, st);         // multiplies the noisy latent
      pack(wf, 256, 0, 0, src + 512, d, 256, in, 1, ROW_IDENT, 1, st);   // multiplies the mixture features
    });
  }
  reg_f32(e, "proj.bias", {d}, &e->proj_b);
  reg_linear(e, "memory_proj.weight", d, c.text_dim, &e->wmem);
  reg_f32(e, "memory_proj.bias", {d}, &e->mem_b);
  e->wvid = e->wpool.alloc<bf16>((int64_t)d * c.vision_dim, true);
  {
    bf16* wv = e->wvid;
    const int vd = c.vision_dim;
    reg(e, "align_masked_video.conv.weight", {d, vd, 1}, [=](const float* src, cudaStream_t st) {
      pack(wv, vd, 0, 0, src, d, vd, vd, 1, ROW_IDENT, 1, st);
    });
  }
  reg_f32(e, "align_masked_video.conv.bias", {d}, &e->vid_b);
  reg_f32(e, "align_masked_video.layer_norm.weight", {d}, &e->vid_ln_w);
  reg_f32(e, "align_masked_video.layer_norm.bias", {d}, &e->vid_ln_b);
  reg_f32(e, "align_masked_video.gate", {1}, &e->vid_gate);
  reg_f32(e, "embed_anchors.embed.weight", {c.n_anchor_tokens, c.anchor_dim}, &e->anchor_embed);
  reg_f32(e, "embed_anchors.proj.weight", {d, c.anchor_dim}, &e->anchor_proj);
  reg_f32(e, "embed_anchors.gate", {1}, &e->anchor_gate);
  e->vid_const = e->wpool.alloc<float>(d, true);
  e->anchor_table = e->wpool.alloc<float>((int64_t)c.n_anchor_tokens * d, true);
  // ---- DiT prologue / epilogue ----
  for (int b = 0; b < 2; ++b) {
    const std::string p = fmt("transformer.x_embedder.block.block%d", b + 1);
    reg_f32(e, p + ".groupnorm.weight", {d}, &e->xe_gn_w[b]);
    reg_f32(e, p + ".groupnorm.bias", {d}, &e->xe_gn_b[b]);
    e->xe_w[b] = e->wpool.alloc<bf16>((int64_t)d * 3 * d, true);
    bf16* w = e->xe_w[b];
    reg(e, p + ".project.weight", {d, d, 3}, [=](const float* src, cudaStream_t st) {
      for (int k = 0; k < 3; ++k) pack(w, 3LL * d, 0, (long long)k * d, src + k, d, d, 3LL * d, 3, ROW_IDENT, 1, st);
    });
    reg_f32(e, p + ".project.bias", {d}, &e->xe_b[b]);
  }
  e->t_w13 = e->wpool.alloc<bf16>((int64_t)2 * d * 256, true);
  reg_linear(e, "transformer.t_embedder.projection.w1.weight", d, 256, nullptr, ROW_SWIGLU_A, 1, e->t_w13, 0, 256);
  reg_linear(e, "transformer.t_embedder.projection.w3.weight", d, 256, nullptr, ROW_SWIGLU_B, 1, e->t_w13, 0, 256);
  reg_linear(e, "transformer.t_embedder.projection.w2.weight", d, d, &e->t_w2);
  reg_linear(e, "transformer.t_block.weight", 6 * d, d, &e->tb_w);
  reg_f32(e, "transformer.t_block.bias", {6 * d}, &e->tb_b);
  e->y_w13 = e->wpool.alloc<bf16>((int64_t)2 * d * d, true);
  reg_linear(e, "transformer.y_embedder.projection.w1.weight", d, d, nullptr, ROW_SWIGLU_A, 1, e->y_w13, 0, d);
  reg_linear(e, "transformer.y_embedder.projection.w3.weight", d, d, nullptr, ROW_SWIGLU_B, 1, e->y_w13, 0, d);
  reg_linear(e, "transformer.y_embedder.projection.w2.weight", d, d, &e->y_w2);
  reg_f32(e, "transformer.norm.weight", {d}, &e->final_norm);
  reg_linear(e, "transformer.output.weight", c.out_channels, d, &e->w_out);
  reg_f32(e, "transformer.final_layer_scale_shift_table", {2, d}, &e->final_table);
  // ---- DiT layers ----
  e->norm_w_all = e->wpool.alloc<float>((int64_t)2 * L * d, true);
  e->tables = e->wpool.alloc<float>((int64_t)L * 6 * d, true);
  e->wkv_c_all = e->wpool.alloc<bf16>((int64_t)L * 2 * d * d, true);   // all layers' cross wk|wv: one GEMM per evaluation
  e->kn_c_all = e->wpool.alloc<float>((int64_t)L * 128, true);
  e->layers.resize(L);
  for (int l = 0; l < L; ++l) {
    LayerW& W = e->layers[l];
    const std::string p = S("transformer.layers.%d", l);
    W.wqkv = e->wpool.alloc<bf16>((int64_t)3 * d * d, true);
    reg_linear(e, p + ".attention.wq.weight", d, d, nullptr, ROW_HEADS, H, W.wqkv, 0, d);
    reg_linear(e, p + ".attention.wk.weight", d, d, nullptr, ROW_HEADS, H, W.wqkv, d, d);
    reg_linear(e, p + ".attention.wv.weight", d, d, nullptr, ROW_HEADS, H, W.wqkv, 2 * d, d);
    reg_linear(e, p + ".attention.wo.weight", d, d, &W.wo);
    reg_f32(e, p + ".attention.q_norm.weight", {128}, &W.qn);
    W.qn_scaled = e->wpool.alloc<float>(128, true);
    reg_f32(e, p + ".attention.k_norm.weight", {128}, &W.kn);
    reg_linear(e, p + ".cross_attention.wq.weight", d, d, &W.wq_c, ROW_HEADS, H);
    W.wkv_c = e->wkv_c_all + (int64_t)l * 2 * d * d;
    reg_linear(e, p + ".cross_attention.wk.weight", d, d, nullptr, ROW_HEADS, H, W.wkv_c, 0, d);
    reg_linear(e, p + ".cross_attention.wv.weight", d, d, nullptr, ROW_HEADS, H, W.wkv_c, d, d);
    reg_linear(e, p + ".cross_attention.wo.weight", d, d, &W.wo_c);
    reg_f32(e, p + ".cross_attention.q_norm.weight", {128}, &W.qn_c);
    W.kn_c = e->kn_c_all + (int64_t)l * 128;
    {
      float* dst = W.kn_c;
      reg(e, p + ".cross_attention.k_norm.weight", {128}, [dst](const float* src, cudaStream_t st) {
        SAB_CUDA(cudaMemcpyAsync(dst, src, 128 * sizeof(float), cudaMemcpyDeviceToDevice, st));
      });
    }
    W.w13 = e->wpool.alloc<bf16>((int64_t)2 * hid * d, true);
    reg_linear(e, p + ".feed_forward.w1.weight", hid, d, nullptr, ROW_SWIGLU_A, 1, W.w13, 0, d);
    reg_linear(e, p + ".feed_forward.w3.weight", hid, d, nullptr, ROW_SWIGLU_B, 1, W.w13, 0, d);
    reg_linear(e, p + ".feed_forward.w2.weight", d, hid, &W.w2);
    reg_f32(e, p + ".attention_norm.weight", {d}, &W.attn_norm);
    reg_f32(e, p + ".ffn_norm.weight", {d}, &W.ffn_norm);
    float* tab = e->tables + (int64_t)l * 6 * d;
    reg(e, p + ".scale_shift_table", {6, d}, [=](const float* src, cudaStream_t st) {
      SAB_CUDA(cudaMemcpyAsync(tab, src, 6LL * d * sizeof(float), cudaMemcpyDeviceToDevice, st));
    });
  }
  // ---- codec ----
  const std::string E = "audio_codec.encoder", D = "audio_codec.decoder", Q = "audio_codec.quantizer";
  const int nr = c.codec_n_rates;
  int ch = c.codec_encoder_dim;
  SAB_CHECK(ch % 64 == 0, "codec encoder_dim must be a multiple of 64");
  reg_f32(e, E + ".block.0.weight", {ch, 1, 7}, &e->enc0_w);
  reg_f32(e, E + ".block.0.bias", {ch}, &e->enc0_b);
  e->enc_blocks.resize(nr);
  for (int i = 0; i < nr; ++i) {
    EncBlockW& B = e->enc_blocks[i];
    const int s = c.codec_encoder_rates[i];
    SAB_CHECK(s % 2 == 0, "codec rates must be even");
    B.cin = ch; B.cout = 2 * ch; B.stride = s;
    const std::string p = fmt("%s.block.%d", E.c_str(), i + 1);
    const int dil[3] = {1, 3, 9};
    for (int j = 0; j < 3; ++j) reg_resunit(e, fmt("%s.block.%d", p.c_str(), j), &B.ru[j], ch, dil[j]);
    reg_f32(e, p + ".block.3.alpha", {1, ch, 1}, &B.a_down);
    reg_conv(e, p + ".block.4", &B.down, 2 * ch, ch, 2 * s, s, 1);
    ch *= 2;
  }
  reg_f32(e, fmt("%s.block.%d.alpha", E.c_str(), nr + 1), {1, ch, 1}, &e->enc_final_alpha);
  reg_conv(e, fmt("%s.block.%d", E.c_str(), nr + 2), &e->enc_final, c.codec_latent_dim, ch, 3, 1, 1);
  {
    // in_proj: only the mean half is used (codec.py:68); packed twice so one GEMM writes [.., 2*cz]
    const int cz = c.codec_codebook_dim, ld = c.codec_latent_dim;
    ConvLayer& P = e->in_proj;
    P.cin = ld; P.cout = 2 * cz; P.k = 1;
    P.w = e->wpool.alloc<bf16>((int64_t)2 * cz * ld, true);
    P.bias = e->wpool.alloc<float>(2 * cz, true);
    bf16* w = P.w; float* bptr = P.bias;
    reg(e, Q + ".in_proj.weight", {2 * cz, ld, 1}, [=](const float* src, cudaStream_t st) {
      pack(w, ld, 0, 0, src, cz, ld, ld, 1, ROW_IDENT, 1, st);
      pack(w, ld, cz, 0, src, cz, ld, ld, 1, ROW_IDENT, 1, st);
    });
    reg(e, Q + ".in_proj.bias", {2 * cz}, [=](const float* src, cudaStream_t st) {
      SAB_CUDA(cudaMemcpyAsync(bptr, src, cz * sizeof(float), cudaMemcpyDeviceToDevice, st));
      SAB_CUDA(cudaMemcpyAsync(bptr + cz, src, cz * sizeof(float), cudaMemcpyDeviceToDevice, st));
    });
    reg_conv(e, Q + ".out_proj", &e->out_proj, ld, cz, 1, 1, 1);
  }
  int dch = c.codec_decoder_dim;
  reg_conv(e, D + ".model.0", &e->dec0, dch, c.codec_latent_dim, 7, 1, 1);
  e->dec_blocks.resize(nr);
  for (int i = 0; i < nr; ++i) {
    DecBlockW& B = e->dec_blocks[i];
    const int s = c.codec_decoder_rates[i];
    B.cin = dch; B.cout = dch / 2; B.stride = s;
    const std::string p = fmt("%s.model.%d", D.c_str(), i + 1);
    reg_f32(e, p + ".block.0.alpha", {1, dch, 1}, &B.a_up);
    reg_convT(e, p + ".block.1", &B.up, dch, dch / 2, s);
    const int dil[3] = {1, 3, 9};
    for (int j = 0; j < 3; ++j) reg_resunit(e, fmt("%s.block.%d", p.c_str(), j + 2), &B.ru[j], dch / 2, dil[j]);
    dch /= 2;
  }
  reg_f32(e, fmt("%s.model.%d.alpha", D.c_str(), nr + 1), {1, dch, 1}, &e->dec_final_alpha);
  reg_f32(e, fmt("%s.model.%d.weight", D.c_str(), nr + 2), {1, dch, 7}, &e->dec_last_w);
  reg_f32(e, fmt("%s.model.%d.bias", D.c_str(), nr + 2), {1}, &e->dec_last_b);
}

// =====================================================================================================
// DiT plan: workspace + launch records for one (Bc, T, L)
// =====================================================================================================
struct LayerOps {
  GemmOp qkv, wo, q_c, kv_c, wo_c, w13, w2;
};
// Everything of a DiT evaluation that depends on the evaluation TIME only (transformer.py:482-493, 363-371, 507-509):
// the timestep embedding, t_block, the adaLN tables of every layer, and — for the fused RMSNorm — the column scales
// w*(1+scale) and the biases shift @ W^T.  R rows = one per sequence (sab_dit_forward: every sequence has its own time)
// or one per evaluation of a solve (sab_solve: all sequences share the time, so the 2*n_steps rows are computed ONCE
// per plan instead of inside the ODE loop, and every consumer reads row k with an item stride of 0).
struct TimeState {
  int R = 0;
  float *time = nullptr, *t = nullptr, *t0 = nullptr, *mod = nullptr, *fin = nullptr, *cs = nullptr;
  float *bias_qkv = nullptr, *bias_w13 = nullptr;
  bf16 *tfreq = nullptr, *t_h = nullptr, *t_silu = nullptr, *shift = nullptr;
  GemmOp g_t13, g_t2, g_tb;
  std::vector<GemmOp> g_bias_qkv, g_bias_w13;
  bool valid = false;      // hoisted state: tables match the current weights and step count
  int n_steps = 0;
};

struct DitPlan {
  int B = 0, cand = 1;                  // clips and candidates per clip: Bc = B * cand sequences (candidate-minor)
  int Bc = 0, T = 0, L = 0;
  int64_t M = 0, MB = 0, ML = 0;        // sequence rows Bc*T, clip rows B*T, clip text rows B*L
  float* condB = nullptr;               // clip-level conditioning GEMM output (aliases cond when cand == 1)
  // fused RMSNorm + modulate (gemm_tc.cuh): column scales w*(1+scale) [2NL, Bc, d], bf16 shifts [2NL, Bc, d],
  // per-(row, n-tile, 32-column chunk parity) partial sums of squares [M, ssq_n], per-item biases shift @ W^T
  bool fused_norm = false;
  float* nrm_ssq = nullptr;
  int ssq_n = 0;
  TimeState ts_item;     // per-sequence times (sab_dit_forward), recomputed every evaluation
  TimeState ts_solve;    // one row per evaluation of the ODE grid (sab_solve), computed once
  DevicePool pool;
  // activations
  float *y, *ymid, *cond, *x0, *c1, *h, *mem_base, *time_dev, *vproj;
  bf16 *y_bf, *gn_a, *hb, *xn, *qkv, *att, *qc, *kvc, *u, *mem_in, *y_h, *ymem, *feat_bf, *text_bf, *vid_bf;
  double* gn_partial;
  uint8_t *pad_mask, *text_mask;
  long long *anchor_ids, *anchor_align;
  int n_ids_cap = 0;
  // ops
  GemmOp g_y13, g_y2, g_in, g_xe[2], g_out, g_cond, g_mem, g_vid, g_kvc_all;
  std::vector<LayerOps> lay;
  CUtensorMap tm_att_q, tm_att_kv;   // fused-QKV buffer viewed as (3d cols, T rows, Bc items): box 64x128 / 64x256
  bool att_tc = false;               // wgmma self-attention: attention_tc2 for T <= 256, attention_stream_tc above
  bool xa_fused = false;             // cross-attention folded into the cross.wq GEMM epilogue (L <= XA_MAX_TK)
  // ... and cross.wo folded into the text values (xattn_fold.cuh): cross.wq writes the probabilities xa_p [M, ldu],
  // cross.wo is a K = heads * L GEMM against the clip's Ut[l] [B * d, ldu], computed once per evaluation
  bool xa_fold = false;
  int ldu = 0;
  bf16 *xa_p = nullptr, *ut = nullptr;
  const bf16** wo_c_tab = nullptr;   // [NL] device copy of the layers' cross wo pointers
  double fold_flops = 0, fold_bytes = 0;
  double flops_per_eval = 0;
  // the whole ODE solve (2*n_steps evaluations for midpoint, ~5.9k launches at 24 layers) as one CUDA graph, captured on the second solve
  // of a plan (the first one runs eagerly and configures every kernel's attributes)
  cudaGraphExec_t solve_graph = nullptr;
  int solve_graph_steps = 0;
  int64_t solve_graph_launches = 0;
  int solves = 0;
  int time_steps_uploaded = 0;
  int solve_method = 0;              // SAB_ODE_* of the cached time tables / captured graph
  int64_t time_cap = 0;              // capacity of time_dev (floats)
  float* rk[4] = {nullptr, nullptr, nullptr, nullptr};   // rk4 stage velocities
  int64_t last_use = 0;              // engine plan_clock of the last sab_prepare that selected this plan
  ~DitPlan() { if (solve_graph) cudaGraphExecDestroy(solve_graph); }
};

static void build_time_state(sab_engine* e, DitPlan& p, TimeState& ts, int R) {
  const sab_config& c = e->cfg;
  const int d = c.dim, hid = c.ffn_hidden, NL = c.n_layers;
  DevicePool& w = p.pool;
  ts.R = R;
  ts.time = w.alloc<float>(R);
  ts.t = w.alloc<float>((int64_t)R * d); ts.t0 = w.alloc<float>((int64_t)R * 6 * d);
  ts.mod = w.alloc<float>((int64_t)NL * R * 6 * d); ts.fin = w.alloc<float>((int64_t)R * 2 * d);
  ts.tfreq = w.alloc<bf16>((int64_t)R * 256); ts.t_h = w.alloc<bf16>((int64_t)R * d);
  ts.t_silu = w.alloc<bf16>((int64_t)R * d);
  ts.g_t13 = make_linear("t_embedder.w13", ts.tfreq, R, 256, e->t_w13, 2 * d, 256, EPI_SWIGLU);
  ts.g_t13.P.out_bf16 = ts.t_h; ts.g_t13.P.out_bf16_ld = d;
  ts.g_t2 = make_linear("t_embedder.w2", ts.t_h, R, d, e->t_w2, d, 256, EPI_AFFINE);
  ts.g_t2.P.out_f32 = ts.t; ts.g_t2.P.out_f32_ld = d;
  ts.g_tb = make_linear("t_block", ts.t_silu, R, d, e->tb_w, 6 * d, 256, EPI_AFFINE);
  ts.g_tb.P.bias = e->tb_b; ts.g_tb.P.out_f32 = ts.t0; ts.g_tb.P.out_f32_ld = 6 * d;
  if (p.fused_norm) {
    ts.cs = w.alloc<float>((int64_t)2 * NL * R * d);
    ts.shift = w.alloc<bf16>((int64_t)2 * NL * R * d);
    ts.bias_qkv = w.alloc<float>((int64_t)NL * R * 3 * d);
    ts.bias_w13 = w.alloc<float>((int64_t)NL * R * 2 * hid);
    ts.g_bias_qkv.resize(NL);
    ts.g_bias_w13.resize(NL);
    for (int l = 0; l < NL; ++l) {
      const LayerW& W = e->layers[l];
      // shift @ W^T: [R, d] x [N, d]^T with the SAME packed weights as the main GEMM (so the bias columns line up
      // with its accumulator columns, head permutation and gate/up interleave included).  Weight-streaming (HBM) bound
      // at a handful of rows: 64-column tiles so that every SM pulls a share of the weight
      ts.g_bias_qkv[l] = make_linear("norm.bias.qkv", ts.shift + (int64_t)(2 * l) * R * d, R, d, W.wqkv, 3 * d, 64, EPI_AFFINE);
      ts.g_bias_qkv[l].P.out_f32 = ts.bias_qkv + (int64_t)l * R * 3 * d; ts.g_bias_qkv[l].P.out_f32_ld = 3 * d;
      ts.g_bias_w13[l] = make_linear("norm.bias.w13", ts.shift + (int64_t)(2 * l + 1) * R * d, R, d, W.w13, 2 * hid, 64, EPI_AFFINE);
      ts.g_bias_w13[l].P.out_f32 = ts.bias_w13 + (int64_t)l * R * 2 * hid; ts.g_bias_w13[l].P.out_f32_ld = 2 * hid;
    }
  }
}

// Conditioning (features, text, video, anchors, masks) is per CLIP; the candidates of a clip (model.py:193-203) share it:
// the once-per-call GEMMs and the text path (memory, y_embedder, cross K/V) run on B clips and the per-sequence
// consumers index clip = sequence / cand.  Inside sab_solve every sequence sees the same time, so the text path of
// a clip is the same for all of its candidates; sab_dit_forward is only used with cand == 1.
static std::unique_ptr<DitPlan> build_dit_plan(sab_engine* e, int B, int cand, int T, int L, int n_ids_cap) {
  const int Bc = B * cand;
  const sab_config& c = e->cfg;
  const int d = c.dim, hid = c.ffn_hidden, NL = c.n_layers;
  auto P = std::make_unique<DitPlan>();
  DitPlan& p = *P;
  p.B = B; p.cand = cand; p.Bc = Bc; p.T = T; p.L = L;
  const int64_t M = (int64_t)Bc * T, MB = (int64_t)B * T, ML = (int64_t)B * L;
  p.M = M; p.MB = MB; p.ML = ML;
  SAB_CHECK(T <= e->rope_len, "T=%d exceeds the RoPE table (%d)", T, e->rope_len);
  // the DiT kernels count rows (sequence x frame) in 32-bit integers (dit_eval's M, rmsnorm_mod_kernel,
  // cond_finish_kernel, the GEMM's row indices); element offsets are 64-bit
  SAB_CHECK(M <= INT32_MAX - 256, "%lld DiT rows (B*candidates=%d x T=%d) exceed the 32-bit row index", (long long)M, Bc,
            T);
  DevicePool& w = p.pool;
  p.y = w.alloc<float>(M * 256); p.ymid = w.alloc<float>(M * 256);
  p.cond = w.alloc<float>(M * d); p.x0 = w.alloc<float>(M * d); p.c1 = w.alloc<float>(M * d);
  p.h = w.alloc<float>(M * d); p.vproj = w.alloc<float>(MB * d);
  p.condB = cand == 1 ? p.cond : w.alloc<float>(MB * d);
  p.mem_base = w.alloc<float>(ML * d);
  p.time_dev = w.alloc<float>((int64_t)Bc * 64); p.time_cap = (int64_t)Bc * 64;
  p.y_bf = w.alloc<bf16>(M * 256); p.gn_a = w.alloc<bf16>(M * d); p.hb = w.alloc<bf16>(M * d);
  p.xn = w.alloc<bf16>(M * d); p.qkv = w.alloc<bf16>(M * 3 * d); p.att = w.alloc<bf16>(M * d);
  p.qc = w.alloc<bf16>(M * d); p.kvc = w.alloc<bf16>(ML * 2 * d * NL); p.u = w.alloc<bf16>(M * hid);
  p.mem_in = w.alloc<bf16>(ML * d); p.y_h = w.alloc<bf16>(ML * d); p.ymem = w.alloc<bf16>(ML * d);
  p.feat_bf = w.alloc<bf16>(MB * 256); p.text_bf = w.alloc<bf16>(ML * c.text_dim);
  p.vid_bf = w.alloc<bf16>(MB * c.vision_dim);
  p.gn_partial = w.alloc<double>((int64_t)Bc * GN_CHUNKS * 2);
  p.pad_mask = w.alloc<uint8_t>(MB); p.text_mask = w.alloc<uint8_t>(ML);
  p.fused_norm = !getenv("SAB_NO_FUSED_NORM");
  if (p.fused_norm) {
    p.ssq_n = 2 * ((d + 255) / 256);
    p.nrm_ssq = w.alloc<float>(M * p.ssq_n, true);
  }
  p.n_ids_cap = n_ids_cap;
  p.anchor_ids = w.alloc<long long>((int64_t)B * p.n_ids_cap); p.anchor_align = w.alloc<long long>(MB);

  // ---- once-per-call conditioning GEMMs ----
  p.g_cond = make_linear("cond.proj_feat", p.feat_bf, MB, 256, e->wp_f, d, 256, EPI_AFFINE);
  p.g_cond.P.bias = e->proj_b; p.g_cond.P.out_f32 = p.condB; p.g_cond.P.out_f32_ld = d;
  p.g_mem = make_linear("cond.memory_proj", p.text_bf, ML, c.text_dim, e->wmem, d, 256, EPI_AFFINE);
  p.g_mem.P.bias = e->mem_b; p.g_mem.P.out_f32 = p.mem_base; p.g_mem.P.out_f32_ld = d;
  p.g_vid = make_linear("cond.align_video", p.vid_bf, MB, c.vision_dim, e->wvid, d, 256, EPI_AFFINE);
  p.g_vid.P.bias = e->vid_b; p.g_vid.P.out_f32 = p.vproj; p.g_vid.P.out_f32_ld = d;

  // ---- per-evaluation prologue (the time-only part lives in a TimeState, built on first use) ----
  p.g_y13 = make_linear("y_embedder.w13", p.mem_in, ML, d, e->y_w13, 2 * d, 256, EPI_SWIGLU);
  p.g_y13.P.out_bf16 = p.y_h; p.g_y13.P.out_bf16_ld = d;
  p.g_y2 = make_linear("y_embedder.w2", p.y_h, ML, d, e->y_w2, d, 256, EPI_AFFINE);
  p.g_y2.P.out_bf16 = p.ymem; p.g_y2.P.out_bf16_ld = d;
  p.g_in = make_linear("proj.noisy", p.y_bf, M, 256, e->wp_y, d, 256, EPI_AFFINE);
  p.g_in.P.res = p.cond; p.g_in.P.res_ld = d; p.g_in.P.out_f32 = p.x0; p.g_in.P.out_f32_ld = d;
  for (int b = 0; b < 2; ++b) {
    RunList rl;   // Conv1d k=3, zero padding (1,1): taps t-1, t, t+1  (patcher.py:52-67)
    for (int k = 0; k < 3; ++k) rl.add(0, k - 1, 0, d / 64);
    p.g_xe[b] = make_gemm(b == 0 ? "x_embedder.conv1" : "x_embedder.conv2", seq_view(p.gn_a, Bc, T, d), e->xe_w[b], d,
                          256, 64, EPI_AFFINE, rl);
    p.g_xe[b].P.bias = e->xe_b[b];
    p.g_xe[b].P.out_f32 = b == 0 ? p.c1 : p.h; p.g_xe[b].P.out_f32_ld = d;
    if (b == 1) { p.g_xe[b].P.res = p.x0; p.g_xe[b].P.res_ld = d; }
  }
  // fused RMSNorm: the kernel that last writes h before a norm also emits that norm's GEMM operand h*w*(1+scale) (into
  // xn) and the partial sums of squares; `which` = 2l (attention_norm of layer l) or 2l+1 (ffn_norm)
  auto norm_producer = [&](GemmOp& op, int which) {
    if (!p.fused_norm) return;
    (void)which;                  // colscale (TimeState row) is bound per evaluation in dit_eval
    op.mode = EPI_AFFINE_NORM;
    op.P.gate_div = T;
    op.P.out_scaled = p.xn; op.P.out_scaled_ld = d;
    op.P.ssq_out = p.nrm_ssq; op.P.ssq_ld = p.ssq_n;
  };
  auto norm_consumer = [&](GemmOp& op) {   // ibias (TimeState row) is bound per evaluation in dit_eval
    if (!p.fused_norm) return;
    op.P.ssq_in = p.nrm_ssq; op.P.ssq_n = p.ssq_n; op.P.ssq_inv_dim = 1.0f / (float)d;
    op.P.ibias_div = T;
  };
  norm_producer(p.g_xe[1], 0);
  // ---- layers ----
  p.lay.resize(NL);
  p.xa_fused = (L <= XA_MAX_TK) && !getenv("SAB_NO_FUSED_XATTN");
  p.xa_fold = p.xa_fused && !getenv("SAB_NO_XATTN_FOLD");
  if (p.xa_fold) {
    p.ldu = (c.n_heads * L + 7) / 8 * 8;   // Ut / P row pitch: 16-byte TMA strides
    p.xa_p = w.alloc<bf16>(M * p.ldu);
    p.ut = w.alloc<bf16>((int64_t)NL * B * d * p.ldu);
    std::vector<const bf16*> tab(NL);
    for (int l = 0; l < NL; ++l) tab[l] = e->layers[l].wo_c;
    p.wo_c_tab = w.alloc<const bf16*>(NL);
    SAB_CUDA(cudaMemcpy(p.wo_c_tab, tab.data(), NL * sizeof(const bf16*), cudaMemcpyHostToDevice));
  }
  for (int l = 0; l < NL; ++l) {
    const LayerW& W = e->layers[l];
    LayerOps& o = p.lay[l];
    const long long kv_ld = 2LL * d * NL;            // layer l's K|V live at columns [l*2d, (l+1)*2d) of p.kvc
    bf16* kvc_l = p.kvc + (long long)l * 2 * d;
    o.qkv = make_linear("attention.qkv", p.xn, M, d, W.wqkv, 3 * d, 256, EPI_QKV);
    o.qkv.P.out_bf16 = p.qkv; o.qkv.P.out_bf16_ld = 3 * d;
    o.qkv.P.qnorm_w = W.qn_scaled; o.qkv.P.knorm_w = W.kn; o.qkv.P.n_q_end = d; o.qkv.P.n_k_end = 2 * d;
    o.qkv.P.rope = e->rope; o.qkv.P.rope_T = T; o.qkv.P.use_rope = 1; o.qkv.P.eps = c.norm_eps;
    norm_consumer(o.qkv);
    o.wo = make_linear("attention.wo", p.att, M, d, W.wo, d, 256, EPI_AFFINE);
    o.wo.P.gate_div = T;     // gate rows (adaLN gate_msa / gate_mlp of the TimeState) are bound per evaluation
    o.wo.P.res = p.h; o.wo.P.res_ld = d; o.wo.P.out_f32 = p.h; o.wo.P.out_f32_ld = d;
    o.wo.P.out_bf16 = p.hb; o.wo.P.out_bf16_ld = d;
    o.q_c = make_linear("cross.wq", p.hb, M, d, W.wq_c, d, 256, EPI_QKV);
    o.q_c.P.out_bf16 = p.qc; o.q_c.P.out_bf16_ld = d;
    o.q_c.P.qnorm_w = W.qn_c; o.q_c.P.knorm_w = W.kn_c; o.q_c.P.n_q_end = d; o.q_c.P.n_k_end = d;
    o.q_c.P.rope_T = T; o.q_c.P.use_rope = 0; o.q_c.P.eps = c.norm_eps;
    if (p.xa_fused) {   // epilogue attends to the layer's text K/V and writes the attention output directly
      SAB_CHECK(o.q_c.BN == 256, "fused cross-attention needs BN=256 tiles");
      o.q_c.tag = "cross.wq+attn";
      o.q_c.P.out_bf16 = p.att; o.q_c.P.out_bf16_ld = d;
      o.q_c.P.xa_kv = kvc_l; o.q_c.P.xa_kv_ld = kv_ld; o.q_c.P.xa_v_col0 = d; o.q_c.P.xa_Tk = L;
      o.q_c.P.xa_T = T * cand;   // query rows per K/V item: the cand sequences of a clip attend to the clip's text
      o.q_c.P.xa_mask = p.text_mask;
      o.q_c.P.xa_scale_log2 = (1.0f / sqrtf(128.f)) * 1.4426950408889634f;
      o.q_c.flops += 4.0 * Bc * c.n_heads * (double)T * L * 128;
    }
    if (p.xa_fold) {    // ... its probabilities only: cross.wo multiplies them with the clip's folded values Ut[l]
      o.q_c.P.out_bf16 = nullptr; o.q_c.P.out_bf16_ld = 0;
      o.q_c.P.xa_p = p.xa_p; o.q_c.P.xa_p_ld = p.ldu;
      o.q_c.flops -= 2.0 * Bc * c.n_heads * (double)T * L * 128;   // no P V
      RunList rl;
      rl.add(0, 0, 0, (c.n_heads * L + 63) / 64);
      const bf16* ut_l = p.ut + (int64_t)l * B * d * p.ldu;
      o.wo_c = make_gemm("cross.wo", AView{p.xa_p, (int64_t)c.n_heads * L, T, Bc, p.ldu, (int64_t)T * p.ldu}, ut_l, d,
                         256, 64, EPI_AFFINE, rl);
      set_per_clip_b(o.wo_c, ut_l, (int64_t)c.n_heads * L, p.ldu, d, cand);
    } else {
      o.wo_c = make_linear("cross.wo", p.att, M, d, W.wo_c, d, 256, EPI_AFFINE);
    }
    o.wo_c.P.res = p.h; o.wo_c.P.res_ld = d; o.wo_c.P.out_f32 = p.h; o.wo_c.P.out_f32_ld = d;
    norm_producer(o.wo_c, 2 * l + 1);
    o.w13 = make_linear("ffn.w13", p.xn, M, d, W.w13, 2 * hid, 256, EPI_SWIGLU);
    o.w13.P.out_bf16 = p.u; o.w13.P.out_bf16_ld = hid; o.w13.P.eps = c.norm_eps;
    norm_consumer(o.w13);
    o.w2 = make_linear("ffn.w2", p.u, M, hid, W.w2, d, 256, EPI_AFFINE);
    o.w2.P.gate_div = T;
    o.w2.P.res = p.h; o.w2.P.res_ld = d; o.w2.P.out_f32 = p.h; o.w2.P.out_f32_ld = d;
    if (l + 1 < NL) norm_producer(o.w2, 2 * (l + 1));      // the last layer feeds the final norm (standalone kernel)
  }
  p.g_out = make_linear("output", p.xn, M, d, e->w_out, c.out_channels, 256, EPI_AFFINE);
  // every layer's text K|V in one GEMM per evaluation: [Bc*L, d] x [NL*2d, d]^T, k-norm per layer
  p.g_kvc_all = make_linear("cross.wkv(all layers)", p.ymem, ML, d, e->wkv_c_all, 2 * d * NL, 256, EPI_QKV);
  p.g_kvc_all.P.out_bf16 = p.kvc; p.g_kvc_all.P.out_bf16_ld = 2LL * d * NL;
  p.g_kvc_all.P.qnorm_w = e->kn_c_all; p.g_kvc_all.P.knorm_w = e->kn_c_all;
  p.g_kvc_all.P.n_q_end = 0; p.g_kvc_all.P.n_k_end = d; p.g_kvc_all.P.qkv_period = 2 * d; p.g_kvc_all.P.norm_w_stride = 128;
  p.g_kvc_all.P.rope_T = L; p.g_kvc_all.P.use_rope = 0; p.g_kvc_all.P.eps = c.norm_eps;
  p.att_tc = !getenv("SAB_NO_TC_ATTENTION");
  if (p.att_tc) {   // the streaming kernel (T > 256) reads Q, K and V through the 128-row box
    p.tm_att_q = make_tmap_3d(p.qkv, 3LL * d, T, Bc, 3LL * d, (int64_t)T * 3 * d, 64, 128);
    if (T <= 256) p.tm_att_kv = make_tmap_3d(p.qkv, 3LL * d, T, Bc, 3LL * d, (int64_t)T * 3 * d, 64, 256);
  }

  // algorithmic FLOPs of one evaluation (GEMMs + attention), for roofline reporting
  double f = p.g_kvc_all.flops + p.g_y13.flops + p.g_y2.flops + p.g_in.flops +
             p.g_xe[0].flops + p.g_xe[1].flops + p.g_out.flops;
  for (auto& o : p.lay)
    f += o.qkv.flops + o.wo.flops + o.q_c.flops + o.wo_c.flops + o.w13.flops + o.w2.flops +
         4.0 * Bc * (double)T * T * d + 4.0 * Bc * (double)T * L * d;
  if (p.xa_fold) {   // Wo of every layer read once, V read once, Ut written once
    p.fold_flops = 2.0 * NL * (double)B * d * c.n_heads * L * 128;
    p.fold_bytes = (double)NL * ((double)d * d * 2.0 + (double)ML * d * 2.0 + (double)B * d * p.ldu * 2.0);
    f += p.fold_flops;
  }
  p.flops_per_eval = f;
  e->dit_plan_builds++;
  return P;
}

// Drop resident DiT plans, least recently used first, until at most `keep` remain.  A victim's workspace and graph may
// still be in use by enqueued work on any stream.
static void evict_dit_plans(sab_engine* e, size_t keep) {
  if (e->dit_plans.size() <= keep) return;
  SAB_CUDA(cudaDeviceSynchronize());
  while (e->dit_plans.size() > keep) {
    auto victim = e->dit_plans.begin();
    for (auto it = e->dit_plans.begin(); it != e->dit_plans.end(); ++it)
      if ((*it)->last_use < (*victim)->last_use) victim = it;
    if (victim->get() == e->dit) e->dit = nullptr;
    e->dit_plans.erase(victim);
  }
}

// =====================================================================================================
// DiT evaluation
// =====================================================================================================
template <int V>
static void launch_rmsnorm(const float* x, const float* w, const float* shift, const float* scale, long long mod_ld,
                           int rows_per_item, bf16* out, int M, float eps, int reverse, cudaStream_t st) {
  rmsnorm_mod_kernel<V><<<(M + 7) / 8, 256, 0, st>>>(x, w, shift, scale, mod_ld, rows_per_item, out, M, eps, reverse);
}
static bool rmsnorm_dim_supported(int d) {
  switch (d) {
    case 256: case 512: case 1024: case 1536: case 2048: case 2560: case 2816: case 3072: case 4096: return true;
    default: return false;
  }
}
static void launch_rmsnorm_mod(int d, const float* x, const float* w, const float* shift, const float* scale,
                               long long mod_ld, int rows_per_item, bf16* out, int M, float eps, int reverse,
                               cudaStream_t st) {
  switch (d / 128) {
#define SAB_RN(v) case v: launch_rmsnorm<v>(x, w, shift, scale, mod_ld, rows_per_item, out, M, eps, reverse, st); break;
    SAB_RN(2) SAB_RN(4) SAB_RN(8) SAB_RN(12) SAB_RN(16) SAB_RN(20) SAB_RN(22) SAB_RN(24) SAB_RN(32)
#undef SAB_RN
    default: throw Error(fmt("rmsnorm: unsupported dim %d (add an instantiation)", d));
  }
  SAB_CUDA(cudaGetLastError());
}
static void rmsnorm_mod(sab_engine* e, const float* x, const float* w, const float* shift, const float* scale,
                        long long mod_ld, int rows_per_item, bf16* out, int M, cudaStream_t st, int reverse = 0) {
  const int d = e->cfg.dim;
  mark(e, st, "rmsnorm_mod", 0, (double)M * d * 6.0);
  launch_rmsnorm_mod(d, x, w, shift, scale, mod_ld, rows_per_item, out, M, e->cfg.norm_eps, reverse, st);
}

// GroupNorm(1) + SiLU of `items` slabs of n_per_item floats (C channels innermost) -> bf16; partial holds
// items * GN_CHUNKS * 2 doubles
static void launch_gn_stats(const float* x, int items, long long n_per_item, double* partial, cudaStream_t st) {
  gn_stats_kernel<<<dim3(GN_CHUNKS, items), 256, 0, st>>>(x, n_per_item, partial);
}
static void launch_gn_apply(const float* x, int items, long long n_per_item, int C, const float* gamma, const float* beta,
                            float eps, const double* partial, bf16* y, cudaStream_t st) {
  gn_silu_kernel<<<dim3(64, items), 256, 0, st>>>(x, partial, gamma, beta, C, n_per_item, eps, y);
}

// the engine's attention dispatch: a handful of text tokens go to the HBM-bound warp-per-row kernel, the rest to the
// flash-style one
static bool attention_is_xattn_small(const AttnParams& ap) { return ap.Tk <= XATT_MAX_TK && ap.k != ap.q; }
static void launch_attention(const AttnParams& ap, int items, int heads, cudaStream_t st) {
  ensure_dynamic_smem(reinterpret_cast<const void*>(attention_kernel), ATT_SMEM);
  if (attention_is_xattn_small(ap)) {
    launch_xattn_small(ap, items, heads, st);
  } else {
    dim3 grid((ap.Tq + ATT_BQ - 1) / ATT_BQ, heads, items);
    attention_kernel<<<grid, ATT_THREADS, ATT_SMEM, st>>>(ap);
  }
  SAB_CUDA(cudaGetLastError());
}
static void attention(sab_engine* e, const AttnParams& ap, int items, int heads, cudaStream_t st) {
  const double fl = 4.0 * items * heads * (double)ap.Tq * ap.Tk * 128;
  if (attention_is_xattn_small(ap)) mark(e, st, "sdpa.cross", fl, (double)items * ap.Tq * heads * 128 * 4.0);
  else mark(e, st, ap.k == ap.q ? "sdpa.self" : "sdpa.cross", fl, 0);
  launch_attention(ap, items, heads, st);
}

// algorithmic HBM bytes of one GEMM launch: operands once + every epilogue stream once (what a perfect kernel moves)
static double gemm_bytes(const GemmOp& op) {
  const GemmParams& P = op.P;
  double per_elem = 0;
  if (P.res) per_elem += 4;
  if (P.out_f32) per_elem += 4;
  if (P.out_bf16) per_elem += 2;
  if (P.out_act) per_elem += 2;
  const double n_out = (op.mode == EPI_SWIGLU) ? P.N / 2.0 : (double)P.N;
  return op.in_bytes + op.rows * n_out * per_elem;
}
// wgmma self-attention (attention_tc2.cuh).  shift_log2 < 0 selects the exact two-pass softmax.
static int g_attn_poly = 2;      // SAB_ATTN_POLY=0..4: pairs of every 8 whose exponential runs on the FMA pipe
template <bool kExact, int kPoly, bool kFolded>
static void launch_attention_tc2_inst(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                                      const AttnTc2Params& ap, cudaStream_t st) {
  auto kern = attention_tc2_kernel<kExact, kPoly, kFolded>;
  ensure_dynamic_smem(reinterpret_cast<const void*>(kern), AT2_SMEM);
  kern<<<ap.heads * ap.items, AT2_THREADS, AT2_SMEM, st>>>(tq, tk, tv, ap);
  SAB_CUDA(cudaGetLastError());
}
// variants: exact (two-pass row maximum; shift_log2 < 0), single pass with scale and shift, and `folded`
// (scale already in q, |logit| <= 50: p = 2^s) — the engine's production path
static void launch_attention_tc2(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                                 const AttnTc2Params& ap, bool folded, cudaStream_t st) {
  const bool exact = ap.shift_log2 < 0.f;
  SAB_CHECK(!(exact && folded), "folded softmax needs a logit bound");
#define SAB_AT2(p_) case p_: return exact ? launch_attention_tc2_inst<true, p_, false>(tq, tk, tv, ap, st)   \
                                  : folded ? launch_attention_tc2_inst<false, p_, true>(tq, tk, tv, ap, st)  \
                                           : launch_attention_tc2_inst<false, p_, false>(tq, tk, tv, ap, st);
  switch (g_attn_poly) {
    SAB_AT2(0) SAB_AT2(2) SAB_AT2(3) SAB_AT2(4)
    default: throw Error(fmt("SAB_ATTN_POLY=%d not built (0, 2, 3, 4)", g_attn_poly));
  }
#undef SAB_AT2
}
// wgmma streaming self-attention for T > 256 (attention_stream_tc.cuh).  shift_log2 >= 0: q is already in the log2
// domain and every |logit| <= shift_log2 <= 50 (bounded variant, no running maximum); < 0: exact online softmax.
template <bool kExact, int kPoly>
static void launch_attention_stream_inst(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                                         const AttnTc2Params& ap, cudaStream_t st) {
  auto kern = attention_stream_tc_kernel<kExact, kPoly>;
  ensure_dynamic_smem(reinterpret_cast<const void*>(kern), ATS_SMEM);
  kern<<<ap.heads * ap.items * ((ap.T + 127) / 128), ATS_THREADS, ATS_SMEM, st>>>(tq, tk, tv, ap);
  SAB_CUDA(cudaGetLastError());
}
static void launch_attention_stream(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                                    const AttnTc2Params& ap, cudaStream_t st) {
  const bool exact = ap.shift_log2 < 0.f;
  SAB_CHECK(exact || ap.shift_log2 <= 50.f, "bounded softmax needs a logit bound <= 50 (got %g)", ap.shift_log2);
#define SAB_ATS(p_) case p_: return exact ? launch_attention_stream_inst<true, p_>(tq, tk, tv, ap, st)   \
                                          : launch_attention_stream_inst<false, p_>(tq, tk, tv, ap, st);
  switch (g_attn_poly) {
    SAB_ATS(0) SAB_ATS(2) SAB_ATS(3) SAB_ATS(4)
    default: throw Error(fmt("SAB_ATTN_POLY=%d not built (0, 2, 3, 4)", g_attn_poly));
  }
#undef SAB_ATS
}

// xattn_fold.cuh: every layer's Ut in one launch.  A CTA sweeps the clips in chunks whose Ut rows it holds in shared
// memory; chunks are sized to about 96 KB so that two CTAs share an SM.
constexpr int XF_MAX_SMEM = 200 * 1024;
static void launch_xattn_fold(XaFoldParams fp, int layers, cudaStream_t st) {
  SAB_CHECK(fp.L >= 1 && fp.L <= XA_MAX_TK, "cross.fold: L=%d outside 1..%d", fp.L, XA_MAX_TK);
  SAB_CHECK(fp.heads * 128 == fp.d && fp.d % XF_ROWS == 0, "cross.fold: d=%d must be heads x 128 (heads=%d)", fp.d, fp.heads);
  SAB_CHECK(fp.ldu % 8 == 0 && fp.ldu >= fp.heads * fp.L, "cross.fold: ldu=%d must be a multiple of 8 and >= heads*L=%d",
            fp.ldu, fp.heads * fp.L);
  SAB_CHECK(fp.clips >= 1 && layers >= 1, "cross.fold: empty launch");
  const int clip_bytes = XF_ROWS * fp.ldu * 2;
  const int max_chunk = std::max(1, 96 * 1024 / clip_bytes);
  const int n_chunks = (fp.clips + max_chunk - 1) / max_chunk;
  fp.chunk = (fp.clips + n_chunks - 1) / n_chunks;
  const int smem = fp.chunk * clip_bytes;
  SAB_CHECK(smem <= XF_MAX_SMEM, "cross.fold: %d bytes of shared memory per clip chunk", smem);
  ensure_dynamic_smem(reinterpret_cast<const void*>(xattn_fold_kernel), XF_MAX_SMEM);
  xattn_fold_kernel<<<dim3(fp.d / XF_ROWS, layers), XF_THREADS, smem, st>>>(fp);
  SAB_CUDA(cudaGetLastError());
}

static void gemm(sab_engine* e, const GemmOp& op, cudaStream_t st) {
  mark(e, st, op.tag, op.flops, gemm_bytes(op));
  launch_gemm(op, st);
}
// Serpentine row order.  Every kernel of a DiT layer is row-parallel and streams activations that exceed the 50 MB
// L2 (fp32 residual 180 MB, fused QKV 270 MB, FFN hidden 241 MB at B = 64): a consumer that walks the rows in the
// same direction as its producer finds the first rows evicted.  Alternating the direction from one launch to the
// next makes each kernel start on the rows its producer wrote last, so roughly an L2's worth of its input (and of the
// in-place residual it updates) never travels to HBM.
static bool g_serpentine = true;   // SAB_NO_SERPENTINE=1 disables (A/B)
static void gemm_dir(sab_engine* e, const GemmOp& op, int& dir, cudaStream_t st) {
  GemmOp o2 = op;
  o2.P.reverse_m = g_serpentine ? dir : 0;
  dir ^= 1;
  gemm(e, o2, st);
}

// final-layer variants: out = base + coef * velocity (ODE axpy fused in the output GEMM's epilogue)
struct FinalSpec {
  const float* base;   // nullptr: plain velocity
  float coef;
  float* out_f32;
  bf16* out_bf16;      // next evaluation's GEMM operand (or nullptr)
};

// the time-only part of an evaluation for the R rows of a TimeState (ts.time holds the R times)
// launch shapes of the time-feature and conditioning kernels, shared by the engine and the unit-test seams
static void launch_tfreq(const float* time, int R, bf16* tfreq, cudaStream_t st) {
  tfreq_kernel<<<(R * 256 + 255) / 256, 256, 0, st>>>(time, R, tfreq);
}
static void launch_mem_time(const float* time, int Bc, int cand, int d, int L, const float* mem_base, bf16* mem_in,
                            cudaStream_t st) {
  mem_time_kernel<<<256, 256, 0, st>>>(time, Bc, cand, d, L, mem_base, mem_in);
}
static void launch_build_mod(const float* tables, const float* t0, float* mod, int NL, int R, int d, const float* ftable,
                             const float* t, float* fin, cudaStream_t st) {
  build_mod_kernel<<<512, 256, 0, st>>>(tables, t0, mod, NL, R, d, ftable, t, fin);
}
static void launch_norm_tables(const float* mod, const float* norm_w, int NL, int R, int d, float* cs, bf16* shift,
                               cudaStream_t st) {
  norm_tables_kernel<<<512, 256, 0, st>>>(mod, norm_w, NL, R, d, cs, shift);
}
static void launch_rope_table(float2* rope, int T, int hd, float theta, cudaStream_t st) {
  rope_table_kernel<<<(T * (hd / 2) + 255) / 256, 256, 0, st>>>(rope, T, hd, theta);
}
static void launch_ln_vector(const float* x, const float* w, const float* b, int d, float* y, cudaStream_t st) {
  ln_vector_kernel<<<1, 256, 0, st>>>(x, w, b, d, y);
}
static void launch_small_abt(const float* A, const float* B, float* C, int I, int J, int K, cudaStream_t st) {
  small_abt_kernel<<<(I * J + 255) / 256, 256, 0, st>>>(A, B, C, I, J, K);
}
static void launch_cond_finish(float* cond, const float* cond_clip, int M, int d, int T, int cand, const float* vproj,
                               const float* ln_w, const float* ln_b, const float* vconst, const float* gate_v,
                               const float* anchor_table, const long long* anchor_ids, int n_ids,
                               const long long* anchor_align, const float* gate_a, int video_term, int anchor_term,
                               cudaStream_t st) {
  cond_finish_kernel<<<(M + 7) / 8, 256, 0, st>>>(cond, cond_clip, M, d, T, cand, vproj, ln_w, ln_b, vconst, gate_v,
                                                  anchor_table, anchor_ids, n_ids, anchor_align, gate_a, video_term,
                                                  anchor_term);
}

static void run_time_state(sab_engine* e, DitPlan& p, TimeState& ts, cudaStream_t st) {
  const sab_config& c = e->cfg;
  const int d = c.dim, NL = c.n_layers, R = ts.R;
  mark(e, st, "time_features_kernel");
  launch_tfreq(ts.time, R, ts.tfreq, st);
  gemm(e, ts.g_t13, st);
  gemm(e, ts.g_t2, st);
  mark(e, st, "silu_cast_kernel");
  silu_cast_kernel<<<64, 256, 0, st>>>(ts.t, ts.t_silu, (long long)R * d);
  gemm(e, ts.g_tb, st);
  mark(e, st, "build_mod_kernel");
  launch_build_mod(e->tables, ts.t0, ts.mod, NL, R, d, e->final_table, ts.t, ts.fin, st);
  if (p.fused_norm) {
    mark(e, st, "norm_tables_kernel");
    launch_norm_tables(ts.mod, e->norm_w_all, NL, R, d, ts.cs, ts.shift, st);
    for (int l = 0; l < NL; ++l) {
      gemm(e, ts.g_bias_qkv[l], st);
      gemm(e, ts.g_bias_w13[l], st);
    }
  }
  SAB_CUDA(cudaGetLastError());
}

// One evaluation.  `row` < 0: ts has one row per sequence (per-item adaLN state); `row` >= 0: ts row `row` holds the
// state of this evaluation's time, shared by every sequence (item stride 0).  time_dev: the Bc times (text memory).
static void dit_eval(sab_engine* e, const float* time_dev, const FinalSpec& fs, const TimeState& ts, int row,
                     cudaStream_t st) {
  DitPlan& p = *e->dit;
  const sab_config& c = e->cfg;
  const int d = c.dim, Bc = p.Bc, T = p.T, L = p.L, NL = c.n_layers, H = c.n_heads, cand = p.cand, hid = c.ffn_hidden;
  const int M = (int)p.M;
  const float sl2 = (1.0f / sqrtf(128.f)) * 1.4426950408889634f;
  const int R = ts.R, r0 = row < 0 ? 0 : row;
  const int istride = row < 0 ? 1 : 0;        // per-item tables advance by one row per sequence, shared ones do not
  auto mod_row = [&](int l, int r) { return ts.mod + (((int64_t)l * R + r0) * 6 + r) * d; };
  auto bind_gate = [&](GemmOp& op, int l, int r) { op.P.gate = mod_row(l, r); op.P.gate_ld = istride * 6 * d; };
  auto bind_cs = [&](GemmOp& op, int which) {
    if (p.fused_norm) { op.P.colscale = ts.cs + ((int64_t)which * R + r0) * d; op.P.colscale_ld = (long long)istride * d; }
  };

  mark(e, st, "mem_time_kernel");
  launch_mem_time(time_dev, Bc, cand, d, L, p.mem_base, p.mem_in, st);
  gemm(e, p.g_y13, st);
  gemm(e, p.g_y2, st);
  gemm(e, p.g_in, st);
  // x_embedder (patcher.py:138-164): GN(1) -> SiLU -> conv3, twice, + x
  for (int b = 0; b < 2; ++b) {
    const float* src = b == 0 ? p.x0 : p.c1;
    mark(e, st, "gn_stats_kernel");
    launch_gn_stats(src, Bc, (long long)T * d, p.gn_partial, st);
    mark(e, st, "gn_silu_kernel");
    launch_gn_apply(src, Bc, (long long)T * d, d, e->xe_gn_w[b], e->xe_gn_b[b], 1e-5f, p.gn_partial, p.gn_a, st);
    GemmOp xe = p.g_xe[b];
    if (b == 1) bind_cs(xe, 0);
    gemm(e, xe, st);
  }
  SAB_CUDA(cudaGetLastError());
  gemm(e, p.g_kvc_all, st);
  if (p.xa_fold) {
    XaFoldParams fp{};
    fp.wo = p.wo_c_tab;
    fp.kv = p.kvc; fp.kv_ld = 2LL * d * NL; fp.kv_layer_cols = 2LL * d; fp.v_col0 = d;
    fp.ut = p.ut; fp.ut_layer_stride = (long long)p.B * d * p.ldu; fp.ldu = p.ldu;
    fp.d = d; fp.heads = H; fp.L = L; fp.clips = p.B;
    mark(e, st, "cross.fold", p.fold_flops, p.fold_bytes);
    launch_xattn_fold(fp, NL, st);
  }
  int dir = 1;   // x_embedder.conv2 (the producer of h) walked the rows forwards
  for (int l = 0; l < NL; ++l) {
    const LayerW& W = e->layers[l];
    LayerOps o = p.lay[l];      // by value: the TimeState rows of this evaluation are bound below
    const long long mod_ld = (long long)istride * 6 * d;
    if (!p.fused_norm) {
      rmsnorm_mod(e, p.h, W.attn_norm, mod_row(l, 0), mod_row(l, 1), mod_ld, T, p.xn, M, st, g_serpentine ? dir : 0);
      dir ^= 1;
    } else {
      o.qkv.P.ibias = ts.bias_qkv + ((int64_t)l * R + r0) * 3 * d; o.qkv.P.ibias_ld = (long long)istride * 3 * d;
      o.w13.P.ibias = ts.bias_w13 + ((int64_t)l * R + r0) * 2 * hid; o.w13.P.ibias_ld = (long long)istride * 2 * hid;
      bind_cs(o.wo_c, 2 * l + 1);
      if (l + 1 < NL) bind_cs(o.w2, 2 * (l + 1));
    }
    bind_gate(o.wo, l, 2);
    bind_gate(o.w2, l, 5);
    gemm_dir(e, o.qkv, dir, st);
    AttnParams a{};
    a.q = p.qkv; a.q_ld = 3 * d; a.q_col0 = 0;
    a.k = p.qkv; a.k_ld = 3 * d; a.k_col0 = d;
    a.v = p.qkv; a.v_ld = 3 * d; a.v_col0 = 2 * d;
    a.o = p.att; a.o_ld = d; a.key_mask = p.pad_mask; a.Tq = T; a.Tk = T; a.mask_div = cand;
    a.scale_log2 = 1.f;          // self-attention: log2(e)/sqrt(hd) is folded into q by the QKV epilogue (W.qn_scaled)
    if (p.att_tc) {
      AttnTc2Params tp{};
      tp.o = p.att; tp.o_ld = d;
      tp.key_mask = p.pad_mask; tp.T = T; tp.heads = H; tp.items = Bc; tp.mask_div = cand;
      // the softmax scale is already in q (QKV epilogue, W.qn_scaled): scale 1 for the exact fallback, and with a
      // logit bound the folded single-pass kernel needs neither scale nor shift
      tp.q_col0 = 0; tp.k_col0 = d; tp.v_col0 = 2 * d; tp.scale_log2 = 1.f; tp.shift_log2 = W.att_shift_log2;
      tp.reverse = g_serpentine ? dir : 0;
      dir ^= 1;
      mark(e, st, "sdpa.self", 4.0 * Bc * H * (double)T * T * 128, (double)M * 4.0 * d * 2.0);   // reads q|k|v, writes o (bf16)
      if (T <= 256) launch_attention_tc2(p.tm_att_q, p.tm_att_kv, p.tm_att_kv, tp, W.att_shift_log2 >= 0.f, st);
      else launch_attention_stream(p.tm_att_q, p.tm_att_q, p.tm_att_q, tp, st);
    } else {
      attention(e, a, Bc, H, st);
    }
    gemm_dir(e, o.wo, dir, st);
    gemm_dir(e, o.q_c, dir, st);
    if (!p.xa_fused) {
      AttnParams x{};
      x.q = p.qc; x.q_ld = d; x.q_col0 = 0;
      x.k = p.kvc; x.k_ld = 2LL * d * NL; x.k_col0 = l * 2 * d;
      x.v = p.kvc; x.v_ld = 2LL * d * NL; x.v_col0 = l * 2 * d + d;
      x.o = p.att; x.o_ld = d; x.key_mask = p.text_mask; x.Tq = T; x.Tk = L; x.scale_log2 = sl2;
      x.kv_div = cand; x.mask_div = cand;
      attention(e, x, Bc, H, st);
    }
    gemm_dir(e, o.wo_c, dir, st);
    if (!p.fused_norm) {
      rmsnorm_mod(e, p.h, W.ffn_norm, mod_row(l, 3), mod_row(l, 4), mod_ld, T, p.xn, M, st, g_serpentine ? dir : 0);
      dir ^= 1;
    }
    gemm_dir(e, o.w13, dir, st);
    gemm_dir(e, o.w2, dir, st);
  }
  rmsnorm_mod(e, p.h, e->final_norm, ts.fin + (int64_t)r0 * 2 * d, ts.fin + (int64_t)r0 * 2 * d + d, (long long)istride * 2 * d, T,
              p.xn, M, st);
  GemmOp out = p.g_out;
  out.P.res = fs.base; out.P.res_ld = 256; out.P.alpha = fs.coef;
  out.P.out_f32 = fs.out_f32; out.P.out_f32_ld = 256;
  out.P.out_bf16 = fs.out_bf16; out.P.out_bf16_ld = 256;
  gemm(e, out, st);
}

// =====================================================================================================
// codec plans
// =====================================================================================================
struct CodecStep {
  enum Kind { GEMM, ENC0, DEC_LAST, LATENT_SPLIT } kind = GEMM;
  GemmOp op;
};
struct CodecPlan {
  std::vector<std::unique_ptr<std::string>> tags;   // owned tag strings (profiling labels)
  const char* tag(const std::string& t) { tags.push_back(std::make_unique<std::string>(t)); return tags.back()->c_str(); }
  int items = 0;       // waveforms per chunk
  long long S = 0;     // samples per waveform
  DevicePool pool;
  std::vector<CodecStep> steps;
  // end-point buffers
  float* x_first = nullptr; bf16* a_first = nullptr;     // encoder stage 0
  bf16* z_in = nullptr;                                  // decoder input [items, T, cz] bf16
  bf16* a_last = nullptr;                                // decoder last-stage activated input
  GemmOp* enc_out = nullptr;                             // in_proj (output pointer patched per chunk)
  float* tile_in = nullptr; float* tile_out = nullptr;   // time-tiled clips: one tile's input and output (allocated on first use)
  double flops = 0;
  int64_t last_use = 0;
};
// A few resident plans per direction (ragged traffic alternates between clip lengths / tail chunks): the least
// recently used ones go until at most `keep` are resident (e->max_codec_plans - 1 before a new shape is planned).
static void evict_codec_plans(sab_engine* e, std::map<std::pair<int, long long>, std::unique_ptr<CodecPlan>>& plans,
                              size_t keep) {
  if (plans.size() <= keep) return;
  SAB_CUDA(cudaDeviceSynchronize());          // the victim's workspace may still be in use by enqueued work
  while (plans.size() > keep) {
    auto victim = plans.begin();
    for (auto it = plans.begin(); it != plans.end(); ++it)
      if (it->second->last_use < victim->second->last_use) victim = it;
    plans.erase(victim);
  }
}

static int pick_bn(int N) {
  if (N % 256 == 0) return 256;
  if (N % 192 == 0) return 192;
  if (N % 128 == 0) return 128;
  if (N % 96 == 0) return 96;
  if (N % 64 == 0) return 64;
  throw Error(fmt("codec: no GEMM tile for N=%d", N));
}
static int pick_bk(int cin) {
  if (cin % 64 == 0) return 64;
  if (cin % 32 == 0) return 32;
  throw Error(fmt("codec: channel count %d not a multiple of 32", cin));
}

struct StageBufs { float* x; bf16* a; bf16* mid; };

// Conv1d(c, c, k=7, dilation) 'same' + Snake  ->  Conv1d(c, c, 1) + residual  (+ Snake for the consumer)
// C <= 128: ONE launch — the 1x1 conv runs back to back on the tensor core from the activated tile in shared
// memory (the intermediate never touches HBM); its output goes to the other operand buffer (sb.a / sb.mid swap)
// because neighbouring tiles still read this unit's input through their dilated taps.
static void plan_resunit(CodecPlan& cp, const ResUnitW& R, int items, long long Tn, int C, StageBufs& sb,
                         const float* next_alpha, bool keep_x) {
  const int bk = pick_bk(C), bn = pick_bn(C);
  static const bool no_b2b = getenv("SAB_NO_B2B") != nullptr;
  if (C <= 128 && bn == C && !no_b2b) {
    RunList rl;
    for (int k = 0; k < 7; ++k) rl.add(0, (k - 3) * R.c7.dil, 0, C / bk);
    CodecStep s;
    s.op = make_gemm(cp.tag(fmt("codec.res.b2b.c%d", C)), seq_view(sb.a, items, Tn, C), R.c7.w, C, bn, bk, EPI_AFFINE, rl, 1);
    s.op.b2b = true;
    s.op.tmW = make_tmap_2d(R.c1.w, C, C, C, bk, bn);
    s.op.P.b2b_bias = R.c7.bias; s.op.P.b2b_alpha = R.a1;
    s.op.P.bias = R.c1.bias;
    s.op.P.res = sb.x; s.op.P.res_ld = C;
    if (keep_x) { s.op.P.out_f32 = sb.x; s.op.P.out_f32_ld = C; }
    s.op.P.out_act = sb.mid; s.op.P.out_act_ld = C; s.op.P.snake_alpha = next_alpha;
    s.op.flops += 2.0 * items * (double)Tn * C * C;
    cp.flops += s.op.flops;
    cp.steps.push_back(s);
    std::swap(sb.a, sb.mid);
    return;
  }
  {
    RunList rl;
    for (int k = 0; k < 7; ++k) rl.add(0, (k - 3) * R.c7.dil, 0, C / bk);
    CodecStep s;
    s.op = make_gemm(cp.tag(fmt("codec.res.conv7.c%d", C)), seq_view(sb.a, items, Tn, C), R.c7.w, C, bn, bk, EPI_AFFINE, rl);
    s.op.P.bias = R.c7.bias;
    s.op.P.out_act = sb.mid; s.op.P.out_act_ld = C; s.op.P.snake_alpha = R.a1;
    cp.flops += s.op.flops;
    cp.steps.push_back(s);
  }
  {
    RunList rl;
    rl.add(0, 0, 0, C / bk);
    CodecStep s;
    s.op = make_gemm(cp.tag(fmt("codec.res.conv1.c%d", C)), seq_view(sb.mid, items, Tn, C), R.c1.w, C, bn, bk, EPI_AFFINE, rl);
    s.op.P.bias = R.c1.bias;
    s.op.P.res = sb.x; s.op.P.res_ld = C;
    if (keep_x) { s.op.P.out_f32 = sb.x; s.op.P.out_f32_ld = C; }
    s.op.P.out_act = sb.a; s.op.P.out_act_ld = C; s.op.P.snake_alpha = next_alpha;
    cp.flops += s.op.flops;
    cp.steps.push_back(s);
  }
}

static CodecPlan* get_enc_plan(sab_engine* e, int items, long long S) {
  auto key = std::make_pair(items, S);
  auto it = e->enc_plans.find(key);
  if (it != e->enc_plans.end()) { it->second->last_use = ++e->plan_clock; return it->second.get(); }
  evict_codec_plans(e, e->enc_plans, e->max_codec_plans - 1);
  e->codec_plan_builds++;
  const sab_config& c = e->cfg;
  auto CP = std::make_unique<CodecPlan>();
  CodecPlan& cp = *CP;
  cp.items = items; cp.S = S;
  int C = c.codec_encoder_dim;
  long long Tn = S;
  StageBufs sb{cp.pool.alloc<float>(items * Tn * C), cp.pool.alloc<bf16>(items * Tn * C), cp.pool.alloc<bf16>(items * Tn * C)};
  cp.x_first = sb.x; cp.a_first = sb.a;
  { CodecStep s; s.kind = CodecStep::ENC0; cp.steps.push_back(s); }
  for (int i = 0; i < c.codec_n_rates; ++i) {
    const EncBlockW& B = e->enc_blocks[i];
    for (int j = 0; j < 3; ++j)
      plan_resunit(cp, B.ru[j], items, Tn, C, sb, j < 2 ? B.ru[j + 1].a0 : B.a_down, j < 2);
    // strided Conv1d(C, 2C, k=2s, stride s, pad s/2) over the [Tn/s, s*C] view of the activated stream
    const int s = B.stride, pd = s / 2;
    SAB_CHECK(Tn % s == 0, "encoder length %lld not divisible by rate %d", Tn, s);
    const long long To = Tn / s;
    const int C2 = 2 * C;
    StageBufs nb{cp.pool.alloc<float>(items * To * C2), cp.pool.alloc<bf16>(items * To * C2),
                 cp.pool.alloc<bf16>(items * To * C2)};
    const int bk = 64;
    SAB_CHECK((pd * C) % bk == 0, "encoder stride tap split not BK aligned");
    RunList rl;
    rl.add(0, -1, (s - pd) * C, pd * C / bk);
    rl.add(0, 0, 0, s * C / bk);
    rl.add(0, +1, 0, (s - pd) * C / bk);
    CodecStep st;
    AView av{sb.a, (int64_t)s * C, To, items, (int64_t)s * C, To * s * C};
    st.op = make_gemm(cp.tag(fmt("codec.enc.down.c%d", C)), av, B.down.w, C2, pick_bn(C2), bk, EPI_AFFINE, rl);
    st.op.P.bias = B.down.bias;
    const bool last = (i == c.codec_n_rates - 1);
    st.op.P.out_f32 = nb.x; st.op.P.out_f32_ld = C2;
    st.op.P.out_act = nb.a; st.op.P.out_act_ld = C2;
    st.op.P.snake_alpha = last ? e->enc_final_alpha : e->enc_blocks[i + 1].ru[0].a0;
    cp.flops += st.op.flops;
    cp.steps.push_back(st);
    sb = nb; C = C2; Tn = To;
  }
  {  // Snake (already applied) -> Conv1d(C, latent, k=3, pad 1) -> bf16 for in_proj
    RunList rl;
    for (int k = 0; k < 3; ++k) rl.add(0, k - 1, 0, C / 64);
    bf16* zl = cp.pool.alloc<bf16>(items * Tn * c.codec_latent_dim);
    CodecStep st;
    st.op = make_gemm("codec.enc.final", seq_view(sb.a, items, Tn, C), e->enc_final.w, c.codec_latent_dim,
                      pick_bn(c.codec_latent_dim), 64, EPI_AFFINE, rl);
    st.op.P.bias = e->enc_final.bias;
    st.op.P.out_bf16 = zl; st.op.P.out_bf16_ld = c.codec_latent_dim;
    cp.flops += st.op.flops;
    cp.steps.push_back(st);
    RunList r1;
    r1.add(0, 0, 0, c.codec_latent_dim / 64);
    CodecStep s2;
    s2.op = make_gemm("codec.in_proj", seq_view(zl, items, Tn, c.codec_latent_dim), e->in_proj.w,
                      2 * c.codec_codebook_dim, pick_bn(2 * c.codec_codebook_dim), 64, EPI_AFFINE, r1);
    s2.op.P.bias = e->in_proj.bias;
    s2.op.P.out_f32_ld = 2 * c.codec_codebook_dim;  // out_f32 patched per call
    cp.flops += s2.op.flops;
    cp.steps.push_back(s2);
  }
  cp.enc_out = &cp.steps.back().op;
  cp.last_use = ++e->plan_clock;
  CodecPlan* r = CP.get();
  e->enc_plans[key] = std::move(CP);
  return r;
}

static CodecPlan* get_dec_plan(sab_engine* e, int items, long long T) {
  auto key = std::make_pair(items, T);
  auto it = e->dec_plans.find(key);
  if (it != e->dec_plans.end()) { it->second->last_use = ++e->plan_clock; return it->second.get(); }
  evict_codec_plans(e, e->dec_plans, e->max_codec_plans - 1);
  e->codec_plan_builds++;
  const sab_config& c = e->cfg;
  auto CP = std::make_unique<CodecPlan>();
  CodecPlan& cp = *CP;
  cp.items = items;
  const int cz = c.codec_codebook_dim, ld = c.codec_latent_dim;
  long long Tn = T;
  cp.z_in = cp.pool.alloc<bf16>(items * Tn * cz);
  { CodecStep s; s.kind = CodecStep::LATENT_SPLIT; cp.steps.push_back(s); }
  bf16* e0 = cp.pool.alloc<bf16>(items * Tn * ld);
  {
    RunList rl;
    rl.add(0, 0, 0, cz / 64);
    CodecStep s;
    s.op = make_gemm("codec.out_proj", seq_view(cp.z_in, items, Tn, cz), e->out_proj.w, ld, pick_bn(ld), 64, EPI_AFFINE, rl);
    s.op.P.bias = e->out_proj.bias;
    s.op.P.out_bf16 = e0; s.op.P.out_bf16_ld = ld;
    cp.flops += s.op.flops;
    cp.steps.push_back(s);
  }
  int C = c.codec_decoder_dim;
  bf16* a_cur = cp.pool.alloc<bf16>(items * Tn * C);
  {
    RunList rl;
    for (int k = 0; k < 7; ++k) rl.add(0, k - 3, 0, ld / 64);
    CodecStep s;
    s.op = make_gemm("codec.dec.conv_in", seq_view(e0, items, Tn, ld), e->dec0.w, C, pick_bn(C), 64, EPI_AFFINE, rl);
    s.op.P.bias = e->dec0.bias;
    s.op.P.out_act = a_cur; s.op.P.out_act_ld = C; s.op.P.snake_alpha = e->dec_blocks[0].a_up;
    cp.flops += s.op.flops;
    cp.steps.push_back(s);
  }
  for (int i = 0; i < c.codec_n_rates; ++i) {
    const DecBlockW& B = e->dec_blocks[i];
    const int s = B.stride, Co = B.cout;
    const long long To = Tn * s;
    StageBufs sb{cp.pool.alloc<float>(items * To * Co), cp.pool.alloc<bf16>(items * To * Co),
                 cp.pool.alloc<bf16>(items * To * Co)};
    {
      // ConvTranspose1d(C, Co, k=2s, stride s, pad s/2): output rows viewed as [Tn, s*Co]
      const int bk = pick_bk(C);
      int bn = pick_bn(Co);                       // must divide the tap switch (s/2)*Co and the period s*Co
      while (bn > 64 && (((s / 2) * Co) % bn != 0)) bn = (bn == 256) ? 192 : (bn == 192) ? 128 : (bn == 128) ? 96 : 64;
      RunList rl;
      rl.period = s * Co; rl.sw = (s / 2) * Co;
      rl.add(0, 0, 0, C / bk); rl.add(0, -1, 0, C / bk);
      rl.add(1, 0, 0, C / bk); rl.add(1, +1, 0, C / bk);
      CodecStep st;
      st.op = make_gemm(cp.tag(fmt("codec.dec.up.c%d", C)), seq_view(a_cur, items, Tn, C), B.up.w, s * Co, bn, bk, EPI_AFFINE, rl);
      st.op.P.bias = B.up.bias; st.op.P.bias_mod = Co;
      st.op.P.out_f32 = sb.x; st.op.P.out_f32_ld = (long long)s * Co;
      st.op.P.out_act = sb.a; st.op.P.out_act_ld = (long long)s * Co; st.op.P.snake_alpha = B.ru[0].a0;
      cp.flops += st.op.flops;
      cp.steps.push_back(st);
    }
    const bool last = (i == c.codec_n_rates - 1);
    const float* after = last ? e->dec_final_alpha : e->dec_blocks[i + 1].a_up;
    for (int j = 0; j < 3; ++j) plan_resunit(cp, B.ru[j], items, To, Co, sb, j < 2 ? B.ru[j + 1].a0 : after, j < 2);
    a_cur = sb.a; C = Co; Tn = To;
  }
  cp.a_last = a_cur;
  cp.S = Tn;
  { CodecStep s; s.kind = CodecStep::DEC_LAST; cp.steps.push_back(s); }
  cp.flops += 2.0 * items * (double)Tn * C * 7;
  cp.last_use = ++e->plan_clock;
  CodecPlan* r = CP.get();
  e->dec_plans[key] = std::move(CP);
  return r;
}

sab_engine::~sab_engine() {
  dit = nullptr;
  dit_plans.clear();
  enc_plans.clear();
  dec_plans.clear();
  if (staging) cudaFree(staging);
  if (capture_stream) cudaStreamDestroy(capture_stream);
  for (auto ev : prof_events) cudaEventDestroy(ev);
}

// =====================================================================================================
// C ABI
// =====================================================================================================
#define SAB_API_BEGIN try {
#define SAB_API_BEGIN_E(e) try { SAB_CHECK((e) != nullptr, "null engine"); DeviceGuard _dg((e)->device);
#define SAB_API_END                                   \
  }                                                   \
  catch (const std::exception& ex) {                  \
    g_last_error = ex.what();                         \
    return 1;                                         \
  }                                                   \
  return 0;

extern "C" {

const char* sab_last_error(void) { return g_last_error.c_str(); }
int sab_version(void) { return 1; }

int sab_create(const sab_config* cfg, int device, sab_engine** out) {
  SAB_API_BEGIN
  SAB_CHECK(cfg && out, "null argument");
  int n_dev = 0;
  cudaError_t ce = cudaGetDeviceCount(&n_dev);
  SAB_CHECK(ce == cudaSuccess && n_dev > 0, "no CUDA device: the SAM-Audio GPU path has no CPU fallback (%s)",
            cudaGetErrorString(ce));
  SAB_CHECK(device >= 0 && device < n_dev && device < kMaxDevices, "bad device index %d", device);
  DeviceGuard _dg(device);
  cudaDeviceProp prop;
  SAB_CUDA(cudaGetDeviceProperties(&prop, device));
  SAB_CHECK(prop.major == 9 && prop.minor == 0, "device %d is sm_%d%d; this library is built for sm_90a only", device,
            prop.major, prop.minor);
  // the A/B switches are re-read by every engine: an unset variable restores the default for engines created later
  {
    const char* f = getenv("SAB_FORCE_CG");
    g_force_cg = f ? atoi(f) : 0;
    SAB_CHECK(g_force_cg >= 0 && g_force_cg <= 2, "SAB_FORCE_CG=%s: expected 1 or 2", f);
    f = getenv("SAB_ATTN_POLY");
    g_attn_poly = f ? atoi(f) : 2;
  }
  g_serpentine = getenv("SAB_NO_SERPENTINE") == nullptr;
  SAB_CHECK(cfg->dim % 128 == 0 && cfg->dim / cfg->n_heads == 128, "dim must be n_heads*128");
  SAB_CHECK(cfg->ffn_hidden % 64 == 0, "ffn_hidden must be a multiple of 64");
  SAB_CHECK(cfg->codec_n_rates >= 1 && cfg->codec_n_rates <= 8, "bad codec_n_rates");
  auto* e = new sab_engine();
  e->cfg = *cfg;
  e->device = device;
  try {
    register_weights(e);
    e->rope_len = cfg->max_positions;
    e->rope = reinterpret_cast<float2*>(e->wpool.alloc<float>((int64_t)e->rope_len * 64 * 2));
    launch_rope_table(e->rope, e->rope_len, 128, cfg->rope_theta, 0);
    SAB_CUDA(cudaGetLastError());
    SAB_CUDA(cudaDeviceSynchronize());
  } catch (...) {
    delete e;
    throw;
  }
  *out = e;
  SAB_API_END
}

int sab_destroy(sab_engine* e) {
  SAB_API_BEGIN
  if (e) {
    DeviceGuard _dg(e->device);
    cudaDeviceSynchronize();
    delete e;
  }
  SAB_API_END
}

int sab_load_weight(sab_engine* e, const char* name, const float* data, const int64_t* shape, int ndim, int is_device,
                    void* stream) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e && name && data, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  auto it = e->slots.find(name);
  SAB_CHECK(it != e->slots.end(), "unexpected weight '%s'", name);
  Slot& s = it->second;
  int64_t n = 1, n_expected = 1;
  for (int i = 0; i < ndim; ++i) n *= shape[i];
  for (auto v : s.shape) n_expected *= v;
  std::vector<int64_t> sq_a, sq_b;  // compare with singleton dims squeezed ([1,C,1] alpha == [C])
  for (auto v : s.shape) if (v != 1) sq_a.push_back(v);
  for (int i = 0; i < ndim; ++i) if (shape[i] != 1) sq_b.push_back(shape[i]);
  SAB_CHECK(sq_a == sq_b, "weight '%s': shape mismatch (expected %lld elements, got %lld)", name,
            (long long)n_expected, (long long)n);
  const float* src = data;
  if (!is_device) {
    if (e->staging_elems < n) {
      if (e->staging) { SAB_CUDA(cudaStreamSynchronize(st)); SAB_CUDA(cudaFree(e->staging)); }
      SAB_CUDA(cudaMalloc(&e->staging, n * sizeof(float)));
      e->staging_elems = n;
    }
    SAB_CUDA(cudaMemcpyAsync(e->staging, data, n * sizeof(float), cudaMemcpyHostToDevice, st));
    src = e->staging;
  }
  s.load(src, st);
  if (!is_device) SAB_CUDA(cudaStreamSynchronize(st));  // staging buffer is reused by the next call
  s.loaded = true;
  e->finalized = false;
  for (auto& p : e->dit_plans) p->ts_solve.valid = false;   // hoisted adaLN tables depend on the weights
  SAB_API_END
}

int sab_finalize_weights(sab_engine* e, int allow_missing, char* missing_out, int64_t missing_cap, void* stream) {
  SAB_API_BEGIN_E(e)
  cudaStream_t st = (cudaStream_t)stream;
  std::string missing, all_missing;
  int n_missing = 0;
  for (auto& kv : e->slots)
    if (!kv.second.loaded) {
      if (n_missing++ < 8) missing += kv.first + " ";
      all_missing += kv.first + "\n";
    }
  SAB_CHECK(n_missing == 0 || allow_missing, "Missing keys (%d): %s", n_missing, missing.c_str());
  if (missing_out && missing_cap > 0) {
    const size_t n = std::min<size_t>(all_missing.size(), (size_t)missing_cap - 1);
    memcpy(missing_out, all_missing.data(), n);
    missing_out[n] = 0;
  }
  const int d = e->cfg.dim;
  // constant video term for text-only prompts: LayerNorm(conv bias)   (SURVEY App. A.9)
  launch_ln_vector(e->vid_b, e->vid_ln_w, e->vid_ln_b, d, e->vid_const, st);
  // anchor table: embed [n,128] @ proj^T [128,d]
  const int n = e->cfg.n_anchor_tokens;
  launch_small_abt(e->anchor_embed, e->anchor_proj, e->anchor_table, n, d, e->cfg.anchor_dim, st);
  SAB_CUDA(cudaGetLastError());
  SAB_CUDA(cudaStreamSynchronize(st));
  for (size_t l = 0; l < e->layers.size(); ++l) {
    SAB_CUDA(cudaMemcpyAsync(e->norm_w_all + (2 * l) * d, e->layers[l].attn_norm, d * sizeof(float), cudaMemcpyDeviceToDevice, st));
    SAB_CUDA(cudaMemcpyAsync(e->norm_w_all + (2 * l + 1) * d, e->layers[l].ffn_norm, d * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  SAB_CUDA(cudaStreamSynchronize(st));
  // self-attention logit bound per layer (see LayerW::att_shift_log2).  The single-pass softmax subtracts this
  // constant instead of the row maximum; it is used only while even a row whose keys are all anti-aligned keeps
  // its largest probability above 2^-100 (2 x shift <= 100), otherwise the layer runs the exact two-pass variant.
  for (auto& W : e->layers) {
    float qn[128], kn[128];
    SAB_CUDA(cudaMemcpy(qn, W.qn, sizeof(qn), cudaMemcpyDeviceToHost));
    SAB_CUDA(cudaMemcpy(kn, W.kn, sizeof(kn), cudaMemcpyDeviceToHost));
    float mq = 0.f, mk = 0.f;
    for (int i = 0; i < 128; ++i) { mq = fmaxf(mq, fabsf(qn[i])); mk = fmaxf(mk, fabsf(kn[i])); }
    const float sl2 = (1.0f / sqrtf(128.f)) * 1.4426950408889634f;
    for (int i = 0; i < 128; ++i) qn[i] *= sl2;
    SAB_CUDA(cudaMemcpy(W.qn_scaled, qn, sizeof(qn), cudaMemcpyHostToDevice));
    const float bound = sqrtf(128.f) * mq * mk * 1.4426950408889634f * 1.02f + 0.25f;   // + bf16 rounding of q, k
    W.att_shift_log2 = (std::isfinite(bound) && bound <= 50.f && !getenv("SAB_ATTN_EXACT")) ? bound : -1.f;
  }
  e->finalized = true;
  SAB_API_END
}

int sab_prepare(sab_engine* e, int B, int candidates, int T, int L, const float* features, const float* text_features,
                const uint8_t* text_mask, const float* video_features, const int64_t* anchor_ids, int n_ids,
                const int64_t* anchor_alignment, const uint8_t* audio_pad_mask, int flags, void* stream) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e->finalized, "weights not finalized");
  SAB_CHECK(B > 0 && candidates > 0 && T > 0 && L > 0, "bad shape");
  SAB_CHECK(features && text_mask && audio_pad_mask, "null argument");
  const bool no_text = (flags & SAB_PREP_NO_TEXT) != 0, no_anchor = (flags & SAB_PREP_NO_ANCHORS) != 0;
  SAB_CHECK(no_text ? L == 1 : text_features != nullptr, "text_features missing (or SAB_PREP_NO_TEXT with L != 1)");
  SAB_CHECK(no_anchor || (anchor_ids && anchor_alignment && n_ids > 0), "anchor tensors missing");
  cudaStream_t st = (cudaStream_t)stream;
  DitPlan* sel = nullptr;
  for (auto& q : e->dit_plans)
    if (q->B == B && q->cand == candidates && q->T == T && q->L == L) sel = q.get();
  if (!sel || n_ids > sel->n_ids_cap) {
    SAB_CUDA(cudaStreamSynchronize(st));
    e->dit = nullptr;                                  // until the new plan exists
    if (sel) {                                         // too small an anchor-id table: this shape is planned anew
      sel->last_use = -1;
      evict_dit_plans(e, e->dit_plans.size() - 1);
    }
    evict_dit_plans(e, e->max_dit_plans - 1);
    // the anchor-id table grows with the longest id list
    e->dit_plans.push_back(build_dit_plan(e, B, candidates, T, L, std::max(64, n_ids)));
    sel = e->dit_plans.back().get();
  }
  sel->last_use = ++e->plan_clock;
  e->dit = sel;
  DitPlan& p = *sel;
  const sab_config& c = e->cfg;
  const int d = c.dim;
  SAB_CHECK(n_ids <= p.n_ids_cap, "too many anchors per clip (%d > %d)", n_ids, p.n_ids_cap);
  const long long M = p.M, MB = p.MB, ML = p.ML;
  SAB_CUDA(cudaMemcpyAsync(p.pad_mask, audio_pad_mask, MB, cudaMemcpyDeviceToDevice, st));
  SAB_CUDA(cudaMemcpyAsync(p.text_mask, text_mask, ML, cudaMemcpyDeviceToDevice, st));
  if (!no_anchor) {
    SAB_CUDA(cudaMemcpyAsync(p.anchor_ids, anchor_ids, (size_t)B * n_ids * 8, cudaMemcpyDeviceToDevice, st));
    SAB_CUDA(cudaMemcpyAsync(p.anchor_align, anchor_alignment, (size_t)MB * 8, cudaMemcpyDeviceToDevice, st));
  }
  mark(e, st, "cast_bf16_kernel");
  cast_bf16_kernel<<<512, 256, 0, st>>>(features, p.feat_bf, MB * 256);
  gemm(e, p.g_cond, st);
  if (no_text) {   // model.py:170-172 with text_features=None: the memory is the time embedding alone
    SAB_CUDA(cudaMemsetAsync(p.mem_base, 0, (size_t)ML * d * sizeof(float), st));
  } else {
    mark(e, st, "cast_bf16_kernel");
    cast_bf16_kernel<<<64, 256, 0, st>>>(text_features, p.text_bf, ML * c.text_dim);
    gemm(e, p.g_mem, st);
  }
  const float* vproj = nullptr;
  if (video_features) {
    mark(e, st, "transpose_cast_kernel");
    transpose_cast_kernel<<<1024, 256, 0, st>>>(video_features, c.vision_dim, T, MB * c.vision_dim, p.vid_bf);
    gemm(e, p.g_vid, st);
    vproj = p.vproj;
  }
  mark(e, st, "cond_finish_kernel");
  launch_cond_finish(p.cond, p.condB, (int)M, d, T, candidates, vproj, e->vid_ln_w, e->vid_ln_b, e->vid_const,
                     e->vid_gate, e->anchor_table, p.anchor_ids, n_ids, p.anchor_align, e->anchor_gate,
                     (flags & SAB_PREP_NO_VIDEO_TERM) ? 0 : 1, no_anchor ? 0 : 1, st);
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

int sab_dit_forward(sab_engine* e, const float* noisy, const float* time, float* velocity, void* stream) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e && e->dit, "sab_prepare must be called first");
  SAB_CHECK(e->dit->cand == 1, "sab_dit_forward takes per-sequence times: prepare with candidates == 1");
  cudaStream_t st = (cudaStream_t)stream;
  DitPlan& p = *e->dit;
  mark(e, st, "cast_bf16_kernel");
  cast_bf16_kernel<<<512, 256, 0, st>>>(noisy, p.y_bf, p.M * 256);
  FinalSpec fs{nullptr, 1.f, velocity, nullptr};
  if (p.ts_item.R == 0) build_time_state(e, p, p.ts_item, p.Bc);
  SAB_CUDA(cudaMemcpyAsync(p.ts_item.time, time, (size_t)p.Bc * sizeof(float), cudaMemcpyDeviceToDevice, st));
  run_time_state(e, p, p.ts_item, st);
  dit_eval(e, time, fs, p.ts_item, -1, st);
  SAB_API_END
}

// stage times (fractions of a step) of the fixed-grid solvers torchdiffeq offers and the reference forwards
// `ode_opt` to (model.py:285-290): euler, midpoint, rk4 (torchdiffeq's rk4 is the 3/8 rule)
static int solver_stages(int method, float (&frac)[4]) {
  switch (method) {
    case SAB_ODE_EULER: frac[0] = 0.f; return 1;
    case SAB_ODE_MIDPOINT: frac[0] = 0.f; frac[1] = 0.5f; return 2;
    case SAB_ODE_RK4: frac[0] = 0.f; frac[1] = 1.f / 3.f; frac[2] = 2.f / 3.f; frac[3] = 1.f; return 4;
    default: throw Error(fmt("unknown ODE method %d (0 midpoint, 1 euler, 2 rk4)", method));
  }
}

int sab_solve(sab_engine* e, const float* noise, int n_steps, int method, float* latent, void* stream) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e && e->dit, "sab_prepare must be called first");
  float frac[4];
  const int S = solver_stages(method, frac);
  const int E = S * n_steps;                   // evaluations per solve
  SAB_CHECK(n_steps >= 1 && E <= 128, "n_steps out of range");
  cudaStream_t st = (cudaStream_t)stream;
  DitPlan& p = *e->dit;
  const long long n = p.M * 256;
  // evaluation times (k + frac_s)/n, broadcast over the batch (model.py:280 t.expand); uploaded once per plan
  if (p.time_steps_uploaded != n_steps || p.solve_method != method) {
    std::vector<float> times((size_t)E * p.Bc);
    for (int k = 0; k < n_steps; ++k)
      for (int sg = 0; sg < S; ++sg)
        for (int b = 0; b < p.Bc; ++b) times[(size_t)(S * k + sg) * p.Bc + b] = ((float)k + frac[sg]) / (float)n_steps;
    if (p.time_cap < (int64_t)times.size()) {
      SAB_CUDA(cudaStreamSynchronize(st));
      p.time_dev = p.pool.alloc<float>((int64_t)times.size());
      p.time_cap = (int64_t)times.size();
    }
    SAB_CUDA(cudaMemcpyAsync(p.time_dev, times.data(), times.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    SAB_CUDA(cudaStreamSynchronize(st));  // `times` is a stack-owned host buffer
    p.time_steps_uploaded = n_steps;
  }
  // The adaLN state depends on the evaluation time only and every sequence of a solve shares it: one row per
  // evaluation, computed once per (plan, solver, step count, weights) instead of inside the loop.
  if (p.ts_solve.R != E || p.solve_method != method) {
    if (p.ts_solve.R != 0) SAB_CUDA(cudaStreamSynchronize(st));
    p.ts_solve = TimeState();     // a new grid: new tables (the old buffers stay with the plan's pool)
    build_time_state(e, p, p.ts_solve, E);
  }
  if (!p.ts_solve.valid) {
    std::vector<float> tk((size_t)E);
    for (int k = 0; k < n_steps; ++k)
      for (int sg = 0; sg < S; ++sg) tk[S * k + sg] = ((float)k + frac[sg]) / (float)n_steps;
    SAB_CUDA(cudaMemcpyAsync(p.ts_solve.time, tk.data(), tk.size() * sizeof(float), cudaMemcpyHostToDevice, st));
    SAB_CUDA(cudaStreamSynchronize(st));
    run_time_state(e, p, p.ts_solve, st);
    p.ts_solve.valid = true;
  }
  if (method == SAB_ODE_RK4 && !p.rk[0])
    for (int i = 0; i < 4; ++i) p.rk[i] = p.pool.alloc<float>(n);
  const bool new_method = p.solve_method != method;
  p.solve_method = method;
  SAB_CUDA(cudaMemcpyAsync(p.y, noise, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  auto enqueue = [&](cudaStream_t st) {
    mark(e, st, "cast_bf16_kernel");
    cast_bf16_kernel<<<512, 256, 0, st>>>(p.y, p.y_bf, n);
    const float dt = 1.0f / (float)n_steps;
    auto tm = [&](int ev) { return p.time_dev + (size_t)ev * p.Bc; };
    for (int k = 0; k < n_steps; ++k) {
      if (method == SAB_ODE_MIDPOINT) {
        // f0 = f(t_k, y); y_mid = y + f0*dt/2     |     y += dt * f(t_k + dt/2, y_mid)   (axpy fused in the output GEMM)
        FinalSpec a{p.y, 0.5f * dt, p.ymid, p.y_bf};
        dit_eval(e, tm(2 * k), a, p.ts_solve, 2 * k, st);
        FinalSpec b{p.y, dt, p.y, p.y_bf};
        dit_eval(e, tm(2 * k + 1), b, p.ts_solve, 2 * k + 1, st);
      } else if (method == SAB_ODE_EULER) {
        FinalSpec a{p.y, dt, p.y, p.y_bf};         // y += dt * f(t_k, y)
        dit_eval(e, tm(k), a, p.ts_solve, k, st);
      } else {
        // torchdiffeq rk4 (3/8 rule): k1 = f(t, y); k2 = f(t + dt/3, y + dt k1/3); k3 = f(t + 2dt/3, y + dt (k2 - k1/3));
        // k4 = f(t + dt, y + dt (k1 - k2 + k3)); y += dt (k1 + 3 k2 + 3 k3 + k4) / 8.  The stage inputs need the raw
        // velocities, so they are combined by a small elementwise kernel instead of the output GEMM's epilogue.
        const float c3 = dt / 3.f;
        auto comb = [&](float* out, float a1, float a2, float a3, float a4) {
          mark(e, st, "ode_combine_kernel");
          ode_combine_kernel<<<512, 256, 0, st>>>(p.y, p.rk[0], a1, p.rk[1], a2, p.rk[2], a3, p.rk[3], a4, out, p.y_bf, n);
        };
        for (int sg = 0; sg < 4; ++sg) {
          FinalSpec v{nullptr, 1.f, p.rk[sg], nullptr};
          dit_eval(e, tm(4 * k + sg), v, p.ts_solve, 4 * k + sg, st);
          if (sg == 0) comb(p.ymid, c3, 0.f, 0.f, 0.f);
          else if (sg == 1) comb(p.ymid, -c3, dt, 0.f, 0.f);
          else if (sg == 2) comb(p.ymid, dt, -dt, dt, 0.f);
          else comb(p.y, dt * 0.125f, dt * 0.375f, dt * 0.375f, dt * 0.125f);
        }
      }
    }
  };
  static const bool use_graph = !getenv("SAB_NO_GRAPH");
  const bool graphable = use_graph && !e->prof && p.solves >= 1;
  if (graphable && (!p.solve_graph || p.solve_graph_steps != n_steps || new_method)) {
    if (p.solve_graph) { SAB_CUDA(cudaGraphExecDestroy(p.solve_graph)); p.solve_graph = nullptr; }
    const int64_t launches_before = e->launches;
    cudaGraph_t g = nullptr;
    if (!e->capture_stream) SAB_CUDA(cudaStreamCreateWithFlags(&e->capture_stream, cudaStreamNonBlocking));
    SAB_CUDA(cudaStreamBeginCapture(e->capture_stream, cudaStreamCaptureModeThreadLocal));
    try {
      enqueue(e->capture_stream);
    } catch (...) {
      cudaStreamEndCapture(e->capture_stream, &g);
      if (g) cudaGraphDestroy(g);
      throw;
    }
    SAB_CUDA(cudaStreamEndCapture(e->capture_stream, &g));
    SAB_CUDA(cudaGraphInstantiate(&p.solve_graph, g, 0));
    SAB_CUDA(cudaGraphDestroy(g));
    p.solve_graph_steps = n_steps;
    e->graph_captures++;
    p.solve_graph_launches = e->launches - launches_before;
    e->launches = launches_before;   // counted when the graph is launched
  }
  if (graphable) {
    SAB_CUDA(cudaGraphLaunch(p.solve_graph, st));
    e->launches += p.solve_graph_launches;
  } else {
    enqueue(st);
  }
  p.solves++;
  SAB_CUDA(cudaMemcpyAsync(latent, p.y, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
  SAB_API_END
}

// The codec's two 1-channel end layers (codec_kernels.cuh).  variant: -1 = the engine's choice (the register kernel
// wherever it applies), 0 = the generic kernel, 1 = the register kernel; a variant that cannot take the shape throws.
static bool enc_conv0_reg_ok(int C0) { return C0 >= 4 && C0 % 4 == 0 && 256 % (C0 / 4) == 0; }
static void launch_enc_conv0(int variant, const float* wav, int items, long long S, int C0, const float* w,
                             const float* bias, const float* alpha, float* x_out, bf16* a_out, cudaStream_t st) {
  SAB_CHECK(C0 >= 4 && C0 % 4 == 0, "enc.conv0: C0=%d must be a positive multiple of 4", C0);
  const bool reg = variant < 0 ? enc_conv0_reg_ok(C0) : variant == 1;
  SAB_CHECK(!reg || enc_conv0_reg_ok(C0), "enc.conv0: the register kernel needs C0/4 to divide 256 (C0=%d)", C0);
  if (reg) {
    const long long per_block = (256 / (C0 / 4)) * ENC0_ITER;
    enc_conv0_reg_kernel<<<dim3((unsigned)((S + per_block - 1) / per_block), items), 256, 0, st>>>(
        wav, S, C0, w, bias, alpha, x_out, a_out);
  } else {
    const long long n = S * (C0 / 4);
    enc_conv0_kernel<<<dim3((unsigned)((n + 255) / 256), items), 256, 0, st>>>(wav, S, C0, w, bias, alpha, x_out, a_out);
  }
  SAB_CUDA(cudaGetLastError());
}
static int dec_last_smem(int C) { return ((DEC_LAST_TB + 6) * (C + 2) + 2) * 2 + 7 * C * 4; }
static bool dec_last_reg_ok(int C) { return C == 64 || C == 96 || C == 128; }
static void launch_dec_last(int variant, const bf16* a, int items, long long S, int C, const float* w, const float* bias,
                            float* wav, cudaStream_t st) {
  SAB_CHECK(C >= 2 && C % 2 == 0, "dec.last: C=%d must be even", C);
  const bool reg = variant < 0 ? dec_last_reg_ok(C) : variant == 1;
  SAB_CHECK(!reg || dec_last_reg_ok(C), "dec.last: the register kernel takes C = 64, 96 or 128 (C=%d)", C);
  SAB_CHECK(reg || dec_last_smem(C) <= 48 * 1024, "dec.last: C=%d needs %d B of shared memory (at most 49152)", C,
            dec_last_smem(C));
  if (reg) {
    const dim3 rgrid((unsigned)((S + 32 * DEC_SEG - 1) / (32 * DEC_SEG)), items);
    if (C == 96) dec_last_reg_kernel<3><<<rgrid, 256, 0, st>>>(a, S, w, bias, wav);
    else if (C == 64) dec_last_reg_kernel<2><<<rgrid, 256, 0, st>>>(a, S, w, bias, wav);
    else dec_last_reg_kernel<4><<<rgrid, 256, 0, st>>>(a, S, w, bias, wav);
  } else {
    dec_last_kernel<<<dim3((unsigned)((S + DEC_LAST_TB - 1) / DEC_LAST_TB), items), DEC_LAST_TB, dec_last_smem(C), st>>>(
        a, S, C, w, bias, wav);
  }
  SAB_CUDA(cudaGetLastError());
}

static void run_codec(sab_engine* e, CodecPlan& cp, int items, const float* wav_in, const float* latent_in, int T,
                      float* out, cudaStream_t st) {
  const sab_config& c = e->cfg;
  for (auto& s : cp.steps) {
    switch (s.kind) {
      case CodecStep::ENC0: {
        const int C0 = c.codec_encoder_dim;
        mark(e, st, "codec.enc.conv0", 2.0 * items * (double)cp.S * C0 * 7, (double)items * cp.S * (4.0 + C0 * 6.0));
        launch_enc_conv0(-1, wav_in, items, cp.S, C0, e->enc0_w, e->enc0_b, e->enc_blocks[0].ru[0].a0, cp.x_first,
                         cp.a_first, st);
        break;
      }
      case CodecStep::LATENT_SPLIT: {
        const int cz = c.codec_codebook_dim;
        mark(e, st, "latent_split_kernel");
        latent_split_kernel<<<512, 256, 0, st>>>(latent_in, T, cz, (long long)items * T * cz, cp.z_in);
        break;
      }
      case CodecStep::DEC_LAST: {
        const int C = c.codec_decoder_dim >> c.codec_n_rates;
        mark(e, st, "codec.dec.last", 2.0 * items * (double)cp.S * C * 7, (double)items * cp.S * (4.0 + C * 2.0));
        launch_dec_last(-1, cp.a_last, items, cp.S, C, e->dec_last_w, e->dec_last_b, out, st);
        break;
      }
      default: {
        GemmOp op = s.op;
        op.P.n_items = items;
        if (&s.op == cp.enc_out) op.P.out_f32 = out;
        const long long tiles = (long long)items * op.P.tiles_per_item * op.P.n_tiles_n;
        op.grid = (int)std::min<long long>(tiles, sm_count() / op.cg) * op.cg;
        op.flops = s.op.flops * (double)items / (double)cp.items;
        op.rows = s.op.rows * (double)items / (double)cp.items;
        op.in_bytes = s.op.in_bytes * (double)items / (double)cp.items;   // (the weight share is negligible here)
        gemm(e, op, st);
      }
    }
  }
  SAB_CUDA(cudaGetLastError());
}

// Workspace of one codec item by the planner's constants (fp32 stream + two bf16 operand buffers per stage, 8 B per
// activation element): ~0.56 GB per 10 s clip in the encoder, ~0.85 GB per 10 s waveform in the decoder.
static double codec_item_bytes(long long S_samples, bool decoder) {
  return (double)S_samples / 480000.0 * (decoder ? 0.85e9 : 0.56e9);
}
static double codec_budget() {   // a chunk's workspace stays near 12 GB
  if (const char* b = getenv("SAB_CODEC_CHUNK_BYTES")) return atof(b);   // tests force small chunks and tiles through this
  return 12e9;
}
static int codec_chunk(long long S_samples, bool decoder) {
  const int n = (int)(codec_budget() / codec_item_bytes(S_samples, decoder));
  return n < 1 ? 1 : (n > 64 ? 64 : n);
}

// ---- time tiling of clips that do not fit the budget whole ----
// The codec is local in time (convolutions, Snake, tanh), so an output frame depends on a bounded window of input
// frames.  The window's half-width ("halo", in latent frames) follows from the layer list: walking from the output
// back to the input, a Conv1d(k, dilation) widens the context by (k - 1) / 2 * dilation samples, a stride-s
// Conv1d(k = 2s) reads the input rows -1 .. +1 of its [T / s, s * C] view and a ConvTranspose1d(k = 2s, stride s) the
// input rows -1 .. +1 of each output row.
static long long conv_ctx(long long r, const ConvLayer& L) { return r + (long long)((L.k - 1) / 2) * L.dil; }
static int codec_halo_frames(const sab_engine* e, bool decoder) {
  const sab_config& c = e->cfg;
  long long r = 0;
  if (decoder) {                                     // waveform samples back to latent frames
    r += 3;                                          // dec.last: 7 taps (dec_last_reg_kernel)
    for (int i = c.codec_n_rates - 1; i >= 0; --i) {
      const DecBlockW& B = e->dec_blocks[i];
      for (int j = 2; j >= 0; --j) r = conv_ctx(conv_ctx(r, B.ru[j].c1), B.ru[j].c7);
      r = (r + B.stride - 1) / B.stride + 1;
    }
    return (int)conv_ctx(r, e->dec0);                // out_proj is 1 x 1
  }
  long long hop = 1;                                 // latent frames back to waveform samples
  r = conv_ctx(r, e->enc_final);                     // in_proj is 1 x 1
  for (int i = c.codec_n_rates - 1; i >= 0; --i) {
    const EncBlockW& B = e->enc_blocks[i];
    r = (r + 1) * B.stride;
    for (int j = 2; j >= 0; --j) r = conv_ctx(conv_ctx(r, B.ru[j].c1), B.ru[j].c7);
    hop *= B.stride;
  }
  r += 3;                                            // enc.conv0: 7 taps (enc_conv0_reg_kernel)
  return (int)((r + hop - 1) / hop);
}
// Tiles of Lt latent frames over a clip of T > Lt frames.  Tile {start, w0, w1} is computed over [start, start + Lt)
// and its rows [w0, w1) are kept: at least `halo` computed rows lie between a kept row and an interior tile edge, and
// the first and last tile end at the clip's edges, where the plan's zero fill is the convolution padding as in an
// un-tiled run.  The last tile is right-aligned, so every tile has the plan's length.
struct CodecTile { int start, w0, w1; };
static std::vector<CodecTile> codec_tiles(int T, int Lt, int halo) {
  std::vector<CodecTile> tiles;
  int w0 = 0;
  for (;;) {
    const int start = w0 == 0 ? 0 : w0 - halo;
    if (start + Lt >= T) { tiles.push_back({T - Lt, w0, T}); return tiles; }
    tiles.push_back({start, w0, start + Lt - halo});
    w0 = start + Lt - halo;
  }
}
// tile length in latent frames for a clip that does not fit the budget as `min_items` whole items; 0: run it whole
static int codec_tile_frames(const sab_engine* e, int T, long long hop, bool decoder) {
  const int min_items = decoder ? 2 : 1;
  if (codec_budget() >= min_items * codec_item_bytes((long long)T * hop, decoder)) return 0;
  const int halo = codec_halo_frames(e, decoder);
  int Lt = (int)(codec_budget() / (min_items * codec_item_bytes(hop, decoder)));
  Lt = std::max(Lt, 4 * halo);                       // at least half of a tile is kept
  return Lt < T ? Lt : 0;
}

int sab_encode(sab_engine* e, const float* wav, int B, int64_t S, float* features, void* stream) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e && e->finalized, "weights not finalized");
  cudaStream_t st = (cudaStream_t)stream;
  long long hop = 1;
  for (int i = 0; i < e->cfg.codec_n_rates; ++i) hop *= e->cfg.codec_encoder_rates[i];
  SAB_CHECK(S % hop == 0, "S=%lld must be padded to a multiple of hop=%lld (codec.py:72-78)", (long long)S, hop);
  const long long T = S / hop;
  const int cf = 2 * e->cfg.codec_codebook_dim;
  if (const int Lt = codec_tile_frames(e, (int)T, hop, false)) {
    // one tile at a time through a plan of tile length; the two ends are staged so that the plan runs unchanged
    CodecPlan* cp = get_enc_plan(e, 1, Lt * hop);
    if (!cp->tile_in) { cp->tile_in = cp->pool.alloc<float>(Lt * hop); cp->tile_out = cp->pool.alloc<float>((int64_t)Lt * cf); }
    const auto tiles = codec_tiles((int)T, Lt, codec_halo_frames(e, false));
    for (int b = 0; b < B; ++b)
      for (const CodecTile& t : tiles) {
        SAB_CUDA(cudaMemcpyAsync(cp->tile_in, wav + b * S + t.start * hop, Lt * hop * sizeof(float), cudaMemcpyDeviceToDevice, st));
        run_codec(e, *cp, 1, cp->tile_in, nullptr, Lt, cp->tile_out, st);
        SAB_CUDA(cudaMemcpyAsync(features + (b * T + t.w0) * cf, cp->tile_out + (int64_t)(t.w0 - t.start) * cf,
                                 (int64_t)(t.w1 - t.w0) * cf * sizeof(float), cudaMemcpyDeviceToDevice, st));
      }
  } else {
    const int chunk = std::min(B, codec_chunk(S, false));
    CodecPlan* cp = get_enc_plan(e, chunk, S);
    for (int b0 = 0; b0 < B; b0 += chunk) {
      const int n = std::min(chunk, B - b0);
      run_codec(e, *cp, n, wav + (long long)b0 * S, nullptr, (int)T, features + (long long)b0 * T * cf, st);
    }
  }
  SAB_API_END
}

int sab_decode(sab_engine* e, const float* latent, int Bc, int T, float* wav, void* stream) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e && e->finalized, "weights not finalized");
  cudaStream_t st = (cudaStream_t)stream;
  long long hop = 1;
  for (int i = 0; i < e->cfg.codec_n_rates; ++i) hop *= e->cfg.codec_decoder_rates[i];
  const long long S = (long long)T * hop;
  const int items = 2 * Bc;
  const int cz = e->cfg.codec_codebook_dim;
  if (const int Lt = codec_tile_frames(e, T, hop, true)) {
    // one tile of one clip at a time: the tile's latent rows [Lt, 2 cz] split into the (target, residual) item pair
    // exactly as a whole clip's do
    CodecPlan* cp = get_dec_plan(e, 2, Lt);
    if (!cp->tile_in) { cp->tile_in = cp->pool.alloc<float>((int64_t)Lt * 2 * cz); cp->tile_out = cp->pool.alloc<float>(2 * Lt * hop); }
    const auto tiles = codec_tiles(T, Lt, codec_halo_frames(e, true));
    for (int b = 0; b < Bc; ++b)
      for (const CodecTile& t : tiles) {
        SAB_CUDA(cudaMemcpyAsync(cp->tile_in, latent + ((long long)b * T + t.start) * 2 * cz, (int64_t)Lt * 2 * cz * sizeof(float),
                                 cudaMemcpyDeviceToDevice, st));
        run_codec(e, *cp, 2, nullptr, cp->tile_in, Lt, cp->tile_out, st);
        for (int half = 0; half < 2; ++half)
          SAB_CUDA(cudaMemcpyAsync(wav + (2LL * b + half) * S + t.w0 * hop, cp->tile_out + half * Lt * hop + (t.w0 - t.start) * hop,
                                   (t.w1 - t.w0) * hop * sizeof(float), cudaMemcpyDeviceToDevice, st));
      }
  } else {
    // whole clips per chunk: items (2b, 2b+1) = (target, residual) come from the two halves of latent row b, so a chunk
    // is always an even number of items, at least one clip (a single-item chunk would decode the target half twice)
    int chunk = std::min(items, std::max(2, codec_chunk(S, true) & ~1));
    CodecPlan* cp = get_dec_plan(e, chunk, T);
    for (int i0 = 0; i0 < items; i0 += chunk) {
      const int n = std::min(chunk, items - i0);
      // items (2b, 2b+1) live in latent row b: chunk boundaries are clip boundaries
      run_codec(e, *cp, n, nullptr, latent + (long long)(i0 / 2) * T * 2 * cz, T, wav + (long long)i0 * S, st);
    }
  }
  SAB_API_END
}

int sab_codec_tiling(sab_engine* e, int decoder, int T, int* halo_frames, int* tile_frames) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e->finalized && halo_frames && tile_frames && T > 0, "bad argument");
  long long hop = 1;
  for (int i = 0; i < e->cfg.codec_n_rates; ++i) hop *= decoder ? e->cfg.codec_decoder_rates[i] : e->cfg.codec_encoder_rates[i];
  *halo_frames = codec_halo_frames(e, decoder != 0);
  *tile_frames = codec_tile_frames(e, T, hop, decoder != 0);
  SAB_API_END
}

int64_t sab_launch_count(sab_engine* e, int reset) {
  if (!e) return -1;
  const int64_t v = e->launches;
  if (reset) e->launches = 0;
  return v;
}

int64_t sab_workspace_bytes(sab_engine* e) {
  if (!e) return -1;
  int64_t b = e->wpool.bytes;
  for (auto& p : e->dit_plans) b += p->pool.bytes;
  for (auto& kv : e->enc_plans) b += kv.second->pool.bytes;
  for (auto& kv : e->dec_plans) b += kv.second->pool.bytes;
  for (auto& kv : e->rs_tables) b += kv.second->pool.bytes;
  return b + e->rs_desc_pool.bytes + e->sp_table_pool.bytes + e->sp_desc_pool.bytes;
}

int sab_set_plan_limits(sab_engine* e, int dit_plans, int codec_plans_per_direction) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(dit_plans >= 1 && codec_plans_per_direction >= 1, "plan limits must be >= 1 (got %d, %d)", dit_plans,
            codec_plans_per_direction);
  e->max_dit_plans = (size_t)dit_plans;
  e->max_codec_plans = (size_t)codec_plans_per_direction;
  evict_dit_plans(e, e->max_dit_plans);
  evict_codec_plans(e, e->enc_plans, e->max_codec_plans);
  evict_codec_plans(e, e->dec_plans, e->max_codec_plans);
  SAB_API_END
}

int sab_plan_stats(sab_engine* e, int64_t* dit_plan_builds, int64_t* graph_captures, int64_t* codec_plan_builds,
                   int* dit_plans_resident, int* codec_plans_resident) {
  SAB_API_BEGIN_E(e)
  if (dit_plan_builds) *dit_plan_builds = e->dit_plan_builds;
  if (graph_captures) *graph_captures = e->graph_captures;
  if (codec_plan_builds) *codec_plan_builds = e->codec_plan_builds;
  if (dit_plans_resident) *dit_plans_resident = (int)e->dit_plans.size();
  if (codec_plans_resident) *codec_plans_resident = (int)(e->enc_plans.size() + e->dec_plans.size());
  SAB_API_END
}

int sab_profile(sab_engine* e, int enable, void* stream) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e, "null engine");
  SAB_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  e->prof = enable != 0;
  e->prof_recs.clear();
  SAB_API_END
}

// JSON: {"tag": {"launches": n, "ms": t, "flops": f, "bytes": b}, ...} aggregated since sab_profile(e, 1).
int sab_profile_report(sab_engine* e, char* buf, int64_t cap, void* stream) {
  SAB_API_BEGIN_E(e)
  SAB_CHECK(e && buf && cap > 2, "bad argument");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = e->prof_recs.size();
  std::map<std::string, std::array<double, 4>> agg;
  if (n > 0) {
    if (e->prof_events.size() <= n) {
      cudaEvent_t ev;
      SAB_CUDA(cudaEventCreate(&ev));
      e->prof_events.push_back(ev);
    }
    SAB_CUDA(cudaEventRecord(e->prof_events[n], st));
    SAB_CUDA(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n; ++i) {
      float ms = 0.f;
      SAB_CUDA(cudaEventElapsedTime(&ms, e->prof_events[i], e->prof_events[i + 1]));
      auto& a = agg[e->prof_recs[i].tag];
      a[0] += 1; a[1] += ms; a[2] += e->prof_recs[i].flops; a[3] += e->prof_recs[i].bytes;
    }
  }
  std::string js = "{";
  bool first = true;
  for (auto& kv : agg) {
    js += fmt("%s\"%s\": {\"launches\": %.0f, \"ms\": %.6f, \"flops\": %.6e, \"bytes\": %.6e}", first ? "" : ", ",
              kv.first.c_str(), kv.second[0], kv.second[1], kv.second[2], kv.second[3]);
    first = false;
  }
  js += "}";
  SAB_CHECK((int64_t)js.size() + 1 <= cap, "profile buffer too small (%zu needed)", js.size() + 1);
  memcpy(buf, js.c_str(), js.size() + 1);
  e->prof_recs.clear();
  SAB_API_END
}

// ---- test seams ----
int sab_test_gemm(int M, int N, int K, const void* a_bf16, const void* b_bf16, float* c, int bn, int bk, int cg,
                  void* stream) {
  SAB_API_BEGIN
  RunList rl;
  SAB_CHECK(K % bk == 0, "K must be a multiple of bk");
  rl.add(0, 0, 0, K / bk);
  GemmOp op = make_gemm("test", flat_view((const bf16*)a_bf16, M, K), (const bf16*)b_bf16, N, bn, bk, EPI_AFFINE, rl, cg);
  op.P.out_f32 = c; op.P.out_f32_ld = N;
  launch_gemm(op, (cudaStream_t)stream);
  SAB_API_END
}

// the descriptor's run lists and epilogue fields, copied into the kernel parameters
static void desc_to_params(const sab_test_gemm_desc& d, GemmParams& P) {
  P.N = d.n;
  for (int l = 0; l < 2; ++l) {
    P.n_runs[l] = d.n_runs[l];
    for (int r = 0; r < GEMM_MAX_RUNS; ++r) P.runs[l][r] = KRun{d.runs[l][r].row_shift, d.runs[l][r].a_col, d.runs[l][r].nkb};
  }
  P.n_period = d.n_period; P.n_switch = d.n_switch;
  P.bias = d.bias; P.bias_mod = d.bias_mod;
  P.gate = d.gate; P.gate_ld = d.gate_ld; P.gate_div = d.gate_div;
  P.alpha = d.alpha; P.relu = d.relu;
  P.res = d.res; P.res_ld = d.res_ld;
  P.out_f32 = d.out_f32; P.out_f32_ld = d.out_f32_ld;
  P.out_bf16 = (bf16*)d.out_bf16; P.out_bf16_ld = d.out_bf16_ld;
  P.out_act = (bf16*)d.out_act; P.out_act_ld = d.out_act_ld; P.snake_alpha = d.snake_alpha;
  P.colscale = d.colscale; P.colscale_ld = d.colscale_ld;
  P.out_scaled = (bf16*)d.out_scaled; P.out_scaled_ld = d.out_scaled_ld;
  P.ssq_out = d.ssq_out; P.ssq_ld = d.ssq_ld;
  P.ssq_in = d.ssq_in; P.ssq_n = d.ssq_n; P.ssq_inv_dim = d.ssq_inv_dim;
  P.ibias = d.ibias; P.ibias_ld = d.ibias_ld; P.ibias_div = d.ibias_div;
  P.b2b_bias = d.b2b_bias; P.b2b_alpha = d.b2b_alpha;
  P.qnorm_w = d.qnorm_w; P.knorm_w = d.knorm_w;
  P.n_q_end = d.n_q_end; P.n_k_end = d.n_k_end; P.qkv_period = d.qkv_period; P.norm_w_stride = d.norm_w_stride;
  P.rope = (const float2*)d.rope; P.rope_T = d.rope_T; P.use_rope = d.use_rope; P.eps = d.eps;
  P.xa_kv = (const bf16*)d.xa_kv; P.xa_kv_ld = d.xa_kv_ld; P.xa_v_col0 = d.xa_v_col0; P.xa_Tk = d.xa_Tk; P.xa_T = d.xa_T;
  P.xa_mask = d.xa_mask; P.xa_scale_log2 = d.xa_scale_log2;
  P.xa_p = (bf16*)d.xa_p; P.xa_p_ld = d.xa_p_ld;
  P.b_clip_rows = d.b_clip_rows; P.b_clip_div = d.b_clip_div;
}

int sab_test_gemm_ex(const sab_test_gemm_desc* d, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(d != nullptr, "null descriptor");
  SAB_CHECK(d->struct_bytes == (int32_t)sizeof(sab_test_gemm_desc),
            "sab_test_gemm_desc.struct_bytes=%d but the library's descriptor has %d bytes (header and binding differ)",
            d->struct_bytes, (int)sizeof(sab_test_gemm_desc));
  SAB_CHECK(d->a && d->b && (!d->b2b || d->w1), "null A / B / w1 operand");
  SAB_CHECK(d->a_cols > 0 && d->a_rows > 0 && d->a_items > 0, "empty A view");
  SAB_CHECK(d->grid_ctas >= 0 && d->group_m >= 0, "grid_ctas / group_m must be >= 0 (0: engine default)");
  for (int l = 0; l < 2; ++l)
    SAB_CHECK(d->n_runs[l] >= 0 && d->n_runs[l] <= GEMM_MAX_RUNS, "%d K runs (at most %d)", d->n_runs[l], GEMM_MAX_RUNS);
  const AView A{(const bf16*)d->a, d->a_cols, d->a_rows, d->a_items, d->a_row_pitch ? d->a_row_pitch : d->a_cols,
                d->a_item_pitch};
  RunList rl;
  for (int l = 0; l < 2; ++l)
    for (int r = 0; r < d->n_runs[l]; ++r) rl.add(l, d->runs[l][r].row_shift, d->runs[l][r].a_col, d->runs[l][r].nkb);
  rl.period = d->n_period; rl.sw = d->n_switch;
  // every rule the engine's own launches obey, before any CUDA call
  const int cg = pick_cg(A, d->bn, d->bk, d->cg);
  {
    GemmParams pre;
    memset(&pre, 0, sizeof(pre));
    desc_to_params(*d, pre);
    pre.group_m = d->group_m ? d->group_m : 1;
    pre.reverse_m = d->reverse_m;
    check_gemm("sab_test_gemm_ex", d->bn, d->bk, d->mode, cg, d->b2b != 0, d->grid_ctas ? d->grid_ctas : cg, pre);
  }
  GemmOp op = make_gemm("sab_test_gemm_ex", A, (const bf16*)d->b, d->n, d->bn, d->bk, d->mode, rl, cg);
  desc_to_params(*d, op.P);   // (the tiling fields stay the planner's)
  if (d->group_m) op.P.group_m = d->group_m;
  op.P.reverse_m = d->reverse_m;
  if (d->grid_ctas) op.grid = d->grid_ctas;
  if (d->b_clip_rows > 0) {
    const int64_t ktot = (int64_t)rl.total_kb(0) * d->bk;
    set_per_clip_b(op, (const bf16*)d->b, d->b_cols ? d->b_cols : ktot, d->b_ld ? d->b_ld : ktot, d->b_clip_rows,
                   d->b_clip_div);
  }
  if (d->b2b) {
    op.b2b = true;
    op.tmW = make_tmap_2d(d->w1, d->n, d->n, d->n, d->bk, d->bn);
  }
  launch_gemm(op, (cudaStream_t)stream);
  SAB_API_END
}

int sab_test_xattn_fold(int layers, int clips, int L, int heads, const void* wo_table, const void* kv, int64_t kv_ld,
                        int64_t kv_layer_cols, int v_col0, void* ut, int ldu, int64_t ut_layer_stride, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(wo_table && kv && ut, "null operand");
  SAB_CHECK(ut_layer_stride >= (int64_t)clips * heads * 128 * ldu, "ut_layer_stride=%lld is below clips * d * ldu",
            (long long)ut_layer_stride);
  XaFoldParams fp{};
  fp.wo = (const bf16* const*)wo_table;
  fp.kv = (const bf16*)kv; fp.kv_ld = kv_ld; fp.kv_layer_cols = kv_layer_cols; fp.v_col0 = v_col0;
  fp.ut = (bf16*)ut; fp.ut_layer_stride = ut_layer_stride; fp.ldu = ldu;
  fp.d = heads * 128; fp.heads = heads; fp.L = L; fp.clips = clips;
  launch_xattn_fold(fp, layers, (cudaStream_t)stream);
  SAB_API_END
}

int sab_test_attention(int items, int heads, int Tq, int Tk, const void* q, const void* k, const void* v,
                       const uint8_t* key_mask, void* o, void* stream) {
  SAB_API_BEGIN
  ensure_dynamic_smem(reinterpret_cast<const void*>(attention_kernel), ATT_SMEM);
  AttnParams a{};
  const long long ld = (long long)heads * 128;
  a.q = (const bf16*)q; a.q_ld = ld; a.k = (const bf16*)k; a.k_ld = ld; a.v = (const bf16*)v; a.v_ld = ld;
  a.o = (bf16*)o; a.o_ld = ld; a.key_mask = key_mask; a.Tq = Tq; a.Tk = Tk;
  a.scale_log2 = (1.0f / sqrtf(128.f)) * 1.4426950408889634f;
  if (Tk <= XATT_MAX_TK && k != q) {
    launch_xattn_small(a, items, heads, (cudaStream_t)stream);
  } else {
    dim3 grid((Tq + ATT_BQ - 1) / ATT_BQ, heads, items);
    attention_kernel<<<grid, ATT_THREADS, ATT_SMEM, (cudaStream_t)stream>>>(a);
  }
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

int sab_test_attention_tc2(int items, int heads, int T, const void* q, const void* k, const void* v,
                           const uint8_t* key_mask, void* o, float shift_log2, int poly, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(T <= 256 && T >= 1, "wgmma attention handles 1 <= T <= 256");
  const long long ld = (long long)heads * 128;
  CUtensorMap tq = make_tmap_3d(q, ld, T, items, ld, (int64_t)T * ld, 64, 128);
  CUtensorMap tk = make_tmap_3d(k, ld, T, items, ld, (int64_t)T * ld, 64, 256);
  CUtensorMap tv = make_tmap_3d(v, ld, T, items, ld, (int64_t)T * ld, 64, 256);
  AttnTc2Params tp{};
  tp.o = (bf16*)o; tp.o_ld = ld;
  tp.key_mask = key_mask; tp.T = T; tp.heads = heads; tp.items = items; tp.mask_div = 1;
  tp.q_col0 = tp.k_col0 = tp.v_col0 = 0;
  tp.scale_log2 = (1.0f / sqrtf(128.f)) * 1.4426950408889634f;
  tp.shift_log2 = shift_log2;
  const int saved = g_attn_poly;
  if (poly >= 0) g_attn_poly = poly;
  try {
    // shift_log2 == 0: folded path (the caller passes q already multiplied by log2(e)/sqrt(hd), |logit| <= 50)
    if (shift_log2 == 0.f) tp.shift_log2 = 50.f;
    launch_attention_tc2(tq, tk, tv, tp, shift_log2 == 0.f, (cudaStream_t)stream);
  } catch (...) {
    g_attn_poly = saved;
    throw;
  }
  g_attn_poly = saved;
  SAB_API_END
}

int sab_test_attention_stream(int items, int heads, int T, const void* q, const void* k, const void* v,
                              const uint8_t* key_mask, void* o, float shift_log2, int poly, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(T >= 1 && items >= 1 && heads >= 1, "bad shape");
  const long long ld = (long long)heads * 128;
  CUtensorMap tq = make_tmap_3d(q, ld, T, items, ld, (int64_t)T * ld, 64, 128);
  CUtensorMap tk = make_tmap_3d(k, ld, T, items, ld, (int64_t)T * ld, 64, 128);
  CUtensorMap tv = make_tmap_3d(v, ld, T, items, ld, (int64_t)T * ld, 64, 128);
  AttnTc2Params tp{};
  tp.o = (bf16*)o; tp.o_ld = ld;
  tp.key_mask = key_mask; tp.T = T; tp.heads = heads; tp.items = items; tp.mask_div = 1;
  tp.q_col0 = tp.k_col0 = tp.v_col0 = 0;
  tp.scale_log2 = (1.0f / sqrtf(128.f)) * 1.4426950408889634f;   // exact variant; the bounded one takes q pre-scaled
  tp.shift_log2 = shift_log2 == 0.f ? 50.f : shift_log2;
  const int saved = g_attn_poly;
  if (poly >= 0) g_attn_poly = poly;
  try {
    launch_attention_stream(tq, tk, tv, tp, (cudaStream_t)stream);
  } catch (...) {
    g_attn_poly = saved;
    throw;
  }
  g_attn_poly = saved;
  SAB_API_END
}

// ---- SIMT kernel seams: each launches the engine's own helper (same kernels, grids and variant choice) ----
static bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }

int sab_test_rmsnorm_mod(int M, int d, const float* x, const float* w, const float* shift, const float* scale,
                         int64_t mod_ld, int rows_per_item, float eps, int reverse, void* out, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(x && w && shift && scale && out, "sab_test_rmsnorm_mod: null argument");
  SAB_CHECK(rmsnorm_dim_supported(d), "sab_test_rmsnorm_mod: no instantiation for d=%d (d/128 in 2,4,8,12,16,20,22,24,32)", d);
  SAB_CHECK(M >= 1 && rows_per_item >= 1, "sab_test_rmsnorm_mod: M=%d and rows_per_item=%d must be >= 1", M, rows_per_item);
  SAB_CHECK(mod_ld >= 0 && mod_ld % 4 == 0, "sab_test_rmsnorm_mod: mod_ld=%lld must be a non-negative multiple of 4",
            (long long)mod_ld);
  SAB_CHECK(reverse == 0 || reverse == 1, "sab_test_rmsnorm_mod: reverse=%d must be 0 or 1", reverse);
  SAB_CHECK(aligned16(x) && aligned16(w) && aligned16(shift) && aligned16(scale) && aligned16(out),
            "sab_test_rmsnorm_mod: operands must be 16-byte aligned");
  launch_rmsnorm_mod(d, x, w, shift, scale, (long long)mod_ld, rows_per_item, (bf16*)out, M, eps, reverse,
                     (cudaStream_t)stream);
  SAB_API_END
}

int sab_test_group_norm_silu(int items, int64_t n_per_item, int C, const float* x, const float* gamma,
                             const float* beta, float eps, void* y, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(x && gamma && beta && y, "sab_test_group_norm_silu: null argument");
  SAB_CHECK(items >= 1 && items <= 65535, "sab_test_group_norm_silu: items=%d outside 1..65535", items);
  SAB_CHECK(C >= 4 && C % 4 == 0, "sab_test_group_norm_silu: C=%d must be a positive multiple of 4", C);
  SAB_CHECK(n_per_item >= C && n_per_item % C == 0, "sab_test_group_norm_silu: n_per_item=%lld must be a multiple of C=%d",
            (long long)n_per_item, C);
  SAB_CHECK(aligned16(x) && aligned16(gamma) && aligned16(beta) && aligned16(y),
            "sab_test_group_norm_silu: operands must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  double* partial = nullptr;
  SAB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&partial), (size_t)items * GN_CHUNKS * 2 * sizeof(double), st));
  launch_gn_stats(x, items, (long long)n_per_item, partial, st);
  launch_gn_apply(x, items, (long long)n_per_item, C, gamma, beta, eps, partial, (bf16*)y, st);
  const cudaError_t launched = cudaGetLastError();
  SAB_CUDA(cudaFreeAsync(partial, st));
  SAB_CUDA(launched);
  SAB_API_END
}

int sab_test_time_features(int R, int cand, int d, int n_layers, int L, const float* time, void* tfreq,
                           const float* mem_base, void* mem_in, const float* tables, const float* t0, const float* ftable,
                           const float* t, float* mod, float* fin, const float* norm_w, float* cs, void* shift,
                           void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(R >= 1 && cand >= 1 && R % cand == 0, "sab_test_time_features: R=%d must be a positive multiple of cand=%d",
            R, cand);
  SAB_CHECK(d >= 4 && d % 4 == 0 && n_layers >= 1 && L >= 1,
            "sab_test_time_features: d=%d must be a positive multiple of 4, n_layers=%d and L=%d >= 1", d, n_layers, L);
  SAB_CHECK(time || (!tfreq && !mem_in), "sab_test_time_features: tfreq / mem_in need time");
  SAB_CHECK(!mem_in || mem_base, "sab_test_time_features: mem_in needs mem_base");
  SAB_CHECK(!mod || (tables && t0 && ftable && t && fin), "sab_test_time_features: mod needs tables, t0, ftable, t and fin");
  SAB_CHECK(!cs || (mod && norm_w && shift), "sab_test_time_features: cs needs mod, norm_w and shift");
  SAB_CHECK(aligned16(tables) && aligned16(t0) && aligned16(ftable) && aligned16(t) && aligned16(mod) && aligned16(fin) &&
            aligned16(norm_w) && aligned16(cs) && aligned16(shift),
            "sab_test_time_features: table operands must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  if (tfreq) launch_tfreq(time, R, (bf16*)tfreq, st);
  if (mem_in) launch_mem_time(time, R, cand, d, L, mem_base, (bf16*)mem_in, st);
  if (mod) launch_build_mod(tables, t0, mod, n_layers, R, d, ftable, t, fin, st);
  if (cs) launch_norm_tables(mod, norm_w, n_layers, R, d, cs, (bf16*)shift, st);
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

int sab_test_cond_finish(int B, int cand, int T, int d, float* cond, const float* cond_clip, const float* vproj,
                         const float* ln_w, const float* ln_b, const float* vid_bias, float* vconst, const float* gate_v,
                         const float* anchor_embed, const float* anchor_proj, int n_anchor, int anchor_dim,
                         float* anchor_table, const int64_t* anchor_ids, int n_ids, const int64_t* anchor_align,
                         const float* gate_a, int flags, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(cond && cond_clip && ln_w && ln_b && vid_bias && vconst && gate_v && anchor_embed && anchor_proj &&
            anchor_table && gate_a, "sab_test_cond_finish: null argument");
  SAB_CHECK(B >= 1 && cand >= 1 && T >= 1 && d >= 1, "sab_test_cond_finish: bad shape (B=%d, cand=%d, T=%d, d=%d)", B,
            cand, T, d);
  SAB_CHECK((int64_t)B * cand * T < (1LL << 31) - 8, "sab_test_cond_finish: B * cand * T rows exceed the int range");
  SAB_CHECK((cand == 1) == (cond == cond_clip), "sab_test_cond_finish: cond aliases cond_clip exactly when cand == 1");
  SAB_CHECK(n_anchor >= 1 && anchor_dim >= 1, "sab_test_cond_finish: n_anchor=%d and anchor_dim=%d must be >= 1",
            n_anchor, anchor_dim);
  const bool anchors = (flags & SAB_PREP_NO_ANCHORS) == 0;
  SAB_CHECK(!anchors || (anchor_ids && anchor_align && n_ids >= 1), "sab_test_cond_finish: anchor tensors missing");
  SAB_CHECK((flags & ~(SAB_PREP_NO_VIDEO_TERM | SAB_PREP_NO_ANCHORS)) == 0, "sab_test_cond_finish: unknown flags %d",
            flags);
  cudaStream_t st = (cudaStream_t)stream;
  launch_ln_vector(vid_bias, ln_w, ln_b, d, vconst, st);
  launch_small_abt(anchor_embed, anchor_proj, anchor_table, n_anchor, d, anchor_dim, st);
  launch_cond_finish(cond, cond_clip, B * cand * T, d, T, cand, vproj, ln_w, ln_b, vconst, gate_v, anchor_table,
                     reinterpret_cast<const long long*>(anchor_ids), n_ids,
                     reinterpret_cast<const long long*>(anchor_align), gate_a,
                     (flags & SAB_PREP_NO_VIDEO_TERM) ? 0 : 1, anchors ? 1 : 0, st);
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

int sab_test_rope_table(int T, int hd, float theta, float* out, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(out, "sab_test_rope_table: null argument");
  SAB_CHECK(T >= 1 && hd >= 2 && hd % 2 == 0 && (int64_t)T * (hd / 2) < (1LL << 31) - 256,
            "sab_test_rope_table: bad shape (T=%d, hd=%d)", T, hd);
  SAB_CHECK(theta > 1.f, "sab_test_rope_table: theta=%g must be > 1", theta);
  launch_rope_table(reinterpret_cast<float2*>(out), T, hd, theta, (cudaStream_t)stream);
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

int sab_test_codec_end(int which, int variant, int items, int64_t S, int C, const void* in, const float* w,
                       const float* bias, const float* alpha, float* x_out, void* a_out, float* wav_out, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(which == 0 || which == 1, "sab_test_codec_end: which=%d must be 0 (enc.conv0) or 1 (dec.last)", which);
  SAB_CHECK(variant >= -1 && variant <= 1, "sab_test_codec_end: variant=%d must be -1, 0 or 1", variant);
  SAB_CHECK(items >= 1 && items <= 65535 && S >= 1, "sab_test_codec_end: bad shape (items=%d, S=%lld)", items,
            (long long)S);
  SAB_CHECK(in && w && bias, "sab_test_codec_end: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  if (which == 0) {
    SAB_CHECK(alpha && x_out && a_out, "sab_test_codec_end: enc.conv0 needs alpha, x_out and a_out");
    SAB_CHECK(aligned16(x_out) && ((uintptr_t)a_out & 7) == 0, "sab_test_codec_end: x_out / a_out misaligned");
    SAB_CHECK(S * (C / 4) / 256 < (1LL << 31), "sab_test_codec_end: S=%lld too long for one launch", (long long)S);
    launch_enc_conv0(variant, (const float*)in, items, S, C, w, bias, alpha, x_out, (bf16*)a_out, st);
  } else {
    SAB_CHECK(wav_out, "sab_test_codec_end: dec.last needs wav_out");
    SAB_CHECK(((uintptr_t)in & 7) == 0, "sab_test_codec_end: the bf16 input must be 8-byte aligned");
    launch_dec_last(variant, (const bf16*)in, items, S, C, w, bias, wav_out, st);
  }
  SAB_API_END
}

int sab_test_attention_cross(int items, int heads, int Tq, int Tk, int cand, const void* q, const void* k, const void* v,
                             const uint8_t* key_mask, void* o, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(q && k && v && o, "sab_test_attention_cross: null argument");
  SAB_CHECK(k != q, "sab_test_attention_cross: k == q selects self-attention");
  SAB_CHECK(items >= 1 && items <= 65535 && heads >= 1 && heads <= 65535 && Tq >= 1 && Tk >= 1,
            "sab_test_attention_cross: bad shape (items=%d, heads=%d, Tq=%d, Tk=%d)", items, heads, Tq, Tk);
  SAB_CHECK(cand >= 1 && items % cand == 0, "sab_test_attention_cross: items=%d must be a multiple of cand=%d", items,
            cand);
  SAB_CHECK(aligned16(q) && aligned16(k) && aligned16(v) && aligned16(o), "sab_test_attention_cross: operands must be "
            "16-byte aligned");
  AttnParams a{};
  const long long ld = (long long)heads * 128;
  a.q = (const bf16*)q; a.q_ld = ld; a.k = (const bf16*)k; a.k_ld = ld; a.v = (const bf16*)v; a.v_ld = ld;
  a.o = (bf16*)o; a.o_ld = ld; a.key_mask = key_mask; a.Tq = Tq; a.Tk = Tk;
  a.scale_log2 = (1.0f / sqrtf(128.f)) * 1.4426950408889634f;
  a.kv_div = cand; a.mask_div = cand;
  launch_attention(a, items, heads, (cudaStream_t)stream);
  SAB_API_END
}

// ---- visual prompting: frame pre-processing (vision_kernels.cuh) ----
// tap windows + normalised weights of one axis, fp32 arithmetic of ATen's _compute_indices_min_size_weights_aa
// (cubic a = -1/2, antialias: support and filter stretch by scale = in / out when down-sampling)
struct AaTaps { int taps = 0; std::vector<int> lo, cnt; std::vector<float> w; };
static AaTaps aa_taps(int in_size, int out_size) {
  AaTaps t;
  const float scale = (float)in_size / (float)out_size;
  const float support = scale >= 1.f ? 2.0f * scale : 2.0f;
  const float invscale = scale >= 1.f ? 1.0f / scale : 1.0f;
  t.taps = (int)ceilf(support) * 2 + 1;
  t.lo.resize(out_size); t.cnt.resize(out_size); t.w.assign((size_t)out_size * t.taps, 0.f);
  const float a = -0.5f;
  for (int i = 0; i < out_size; ++i) {
    const float center = scale * ((float)i + 0.5f);
    int lo = (int)(center - support + 0.5f);
    lo = lo < 0 ? 0 : lo;
    int hi = (int)(center + support + 0.5f);
    hi = hi > in_size ? in_size : hi;
    int n = hi - lo;
    n = n < 0 ? 0 : (n > t.taps ? t.taps : n);
    float tot = 0.f;
    float* w = &t.w[(size_t)i * t.taps];
    for (int j = 0; j < n; ++j) {
      float x = fabsf(((float)(j + lo) - center + 0.5f)) * invscale;
      float v;
      if (x < 1.f) v = ((a + 2.f) * x - (a + 3.f)) * x * x + 1.f;
      else if (x < 2.f) v = (((x - 5.f) * x + 8.f) * x - 4.f) * a;
      else v = 0.f;
      w[j] = v;
      tot = tot + v;
    }
    for (int j = 0; j < n; ++j) w[j] = w[j] / tot;
    t.lo[i] = lo; t.cnt[i] = n;
  }
  return t;
}
struct AaTapsDev { int taps; int *lo, *cnt; float* w; };
static AaTapsDev aa_taps_device(int in_size, int out_size) {   // cached per (device, in, out): a few KB each
  static std::map<std::array<int, 3>, AaTapsDev> cache;
  const std::array<int, 3> key = {cur_device(), in_size, out_size};
  auto it = cache.find(key);
  if (it != cache.end()) return it->second;
  const AaTaps h = aa_taps(in_size, out_size);
  AaTapsDev d{h.taps, nullptr, nullptr, nullptr};
  SAB_CUDA(cudaMalloc(&d.lo, out_size * sizeof(int)));
  SAB_CUDA(cudaMalloc(&d.cnt, out_size * sizeof(int)));
  SAB_CUDA(cudaMalloc(&d.w, h.w.size() * sizeof(float)));
  SAB_CUDA(cudaMemcpy(d.lo, h.lo.data(), out_size * sizeof(int), cudaMemcpyHostToDevice));
  SAB_CUDA(cudaMemcpy(d.cnt, h.cnt.data(), out_size * sizeof(int), cudaMemcpyHostToDevice));
  SAB_CUDA(cudaMemcpy(d.w, h.w.data(), h.w.size() * sizeof(float), cudaMemcpyHostToDevice));
  cache[key] = d;
  return d;
}

/* host-only test seam: the evaluation times sab_solve uploads for a solver and step count (no GPU needed) */
int sab_test_solver_grid(int method, int n_steps, int cap, int* n_evals, float* times) {
  SAB_API_BEGIN
  SAB_CHECK(n_evals && times && n_steps >= 1, "bad argument");
  float frac[4];
  const int S = solver_stages(method, frac);
  SAB_CHECK(S * n_steps <= cap, "capacity %d < %d", cap, S * n_steps);
  *n_evals = S * n_steps;
  for (int k = 0; k < n_steps; ++k)
    for (int sg = 0; sg < S; ++sg) times[S * k + sg] = ((float)k + frac[sg]) / (float)n_steps;
  SAB_API_END
}

/* host-only test seam: the tap windows / weights the resize kernels use (no GPU needed) */
int sab_test_aa_taps(int in_size, int out_size, int cap, int* taps, int* lo, int* cnt, float* w) {
  SAB_API_BEGIN
  SAB_CHECK(in_size >= 1 && out_size >= 1 && taps && lo && cnt && w, "bad argument");
  const AaTaps t = aa_taps(in_size, out_size);
  SAB_CHECK(t.taps <= cap, "tap capacity %d < %d", cap, t.taps);
  *taps = t.taps;
  for (int i = 0; i < out_size; ++i) {
    lo[i] = t.lo[i];
    cnt[i] = t.cnt[i];
    for (int j = 0; j < cap; ++j) w[(size_t)i * cap + j] = j < t.taps ? t.w[(size_t)i * t.taps + j] : 0.f;
  }
  SAB_API_END
}

int sab_preprocess_frames(const uint8_t* frames, int n_frames, int H, int W, int out_size, float* workspace, float* out,
                          void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(frames && out && workspace, "null argument");
  SAB_CHECK(n_frames >= 1 && H >= 1 && W >= 1 && out_size >= 1 && W <= 48 * 1024, "bad frame shape");
  cudaStream_t st = (cudaStream_t)stream;
  const AaTapsDev tx = aa_taps_device(W, out_size), ty = aa_taps_device(H, out_size);
  const int planes = n_frames * 3;
  resize_rows_kernel<<<dim3(H, planes), 256, W, st>>>(frames, H, W, out_size, tx.lo, tx.cnt, tx.w, tx.taps, workspace);
  resize_cols_finish_kernel<<<dim3(out_size, planes), 256, 0, st>>>(workspace, H, out_size, ty.lo, ty.cnt, ty.w, ty.taps, out);
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

int sab_blend_windows(const float* win_latent, int n_win, int Tw, const int32_t* win_seq, const int32_t* win_start,
                      const uint8_t* win_flags, int ramp, float* latent, int Bc, int T, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(win_latent && win_seq && win_start && win_flags && latent, "null argument");
  SAB_CHECK(n_win >= 1 && Tw >= 1 && ramp >= 1 && T >= 1, "bad shape (n_win=%d, Tw=%d, ramp=%d, T=%d)", n_win, Tw, ramp, T);
  SAB_CHECK(Bc >= 1 && Bc <= 65535, "Bc=%d outside 1..65535", Bc);
  BlendParams bp{win_latent, win_seq, win_start, win_flags, n_win, Tw, ramp, latent, T};
  const int per_cta = BW_WARPS * BW_FRAMES;
  blend_windows_kernel<<<dim3((T + per_cta - 1) / per_cta, Bc), BW_WARPS * 32, 0, (cudaStream_t)stream>>>(bp);
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

// ---- resampling (resample.cuh) ----
static int64_t floor_div(int64_t a, int64_t b) { return a / b - ((a % b != 0) && ((a < 0) != (b < 0))); }
static int64_t ceil_div(int64_t a, int64_t b) { return -floor_div(-a, b); }

// The polyphase table of torchaudio's sinc_interp_hann design (lowpass_filter_width 6, rolloff 0.99), evaluated in
// float64 and rounded once to fp32.  With base = 0.99 min(o, n) and R = 6 o / base = 600 o / (99 min(o, n)), an exact
// rational, K = 2 ceil(R) + 1 and lo[j] is the first integer i with i / o - j / n >= -R / o; both come from integer
// arithmetic, so no rounding decides which taps a phase has.  w[j][k] = sinc(pi t) cos^2(pi t / 12) base / o with
// t = clamp((lo[j] + k) / o - j / n, +-6 / base) base.
struct ResampleTable { int o = 1, n = 1, K = 1; std::vector<int> lo; std::vector<float> w; };
static bool resample_rate_ok(int r) { return r >= 8000 && r <= 192000; }
static ResampleTable resample_table(int orig, int nw) {
  ResampleTable t;
  if (orig == nw) {                                  // the identity, as in torchaudio: no filter
    t.lo = {0};
    t.w = {1.f};
    return t;
  }
  int64_t a = orig, b = nw;
  while (b) { const int64_t r = a % b; a = b; b = r; }
  const int64_t o = orig / a, n = nw / a, mn = o < n ? o : n;
  const int64_t den = 99 * mn;                       // R = 600 o / den
  t.o = (int)o; t.n = (int)n;
  t.K = (int)(2 * ceil_div(600 * o, den) + 1);
  t.lo.resize(n);
  t.w.resize((size_t)n * t.K);
  const double base = 0.99 * (double)mn, pi = 3.14159265358979323846;
  for (int64_t j = 0; j < n; ++j) {
    // i n den >= j o den - 600 o n
    const int64_t lo = ceil_div(j * o * den - 600 * o * n, n * den);
    t.lo[j] = (int)lo;
    for (int k = 0; k < t.K; ++k) {
      double x = (double)((lo + k) * n - j * o) / ((double)o * (double)n) * base;
      x = x < -6.0 ? -6.0 : (x > 6.0 ? 6.0 : x);
      const double c = cos(x * pi / 12.0);
      const double s = x == 0.0 ? 1.0 : sin(pi * x) / (pi * x);
      t.w[(size_t)j * t.K + k] = (float)(s * (c * c * base / (double)o));
    }
  }
  return t;
}

static const ResampleTableDev& resample_table_dev(sab_engine* e, int orig, int nw) {
  auto& slot = e->rs_tables[{orig, nw}];
  if (!slot) {
    const ResampleTable h = resample_table(orig, nw);
    auto d = std::make_unique<ResampleTableDev>();
    d->o = h.o; d->n = h.n; d->K = h.K;
    d->w = d->pool.alloc<float>((int64_t)h.w.size());
    d->lo = d->pool.alloc<int>((int64_t)h.lo.size());
    std::vector<float> wt(h.w.size());                 // k-major on the device: a warp's phases read adjacent floats
    for (int j = 0; j < h.n; ++j)
      for (int k = 0; k < h.K; ++k) wt[(size_t)k * h.n + j] = h.w[(size_t)j * h.K + k];
    SAB_CUDA(cudaMemcpy(d->w, wt.data(), wt.size() * sizeof(float), cudaMemcpyHostToDevice));
    SAB_CUDA(cudaMemcpy(d->lo, h.lo.data(), h.lo.size() * sizeof(int), cudaMemcpyHostToDevice));
    slot = std::move(d);
  }
  return *slot;
}

int sab_resample_taps(int orig_rate, int new_rate, int64_t cap, int* K, int* lo, float* w) {
  SAB_API_BEGIN
  SAB_CHECK(K, "null argument");
  SAB_CHECK(resample_rate_ok(orig_rate) && resample_rate_ok(new_rate), "rates %d -> %d: both must lie in [8000, 192000]",
            orig_rate, new_rate);
  const ResampleTable t = resample_table(orig_rate, new_rate);
  *K = t.K;
  if (lo) memcpy(lo, t.lo.data(), t.lo.size() * sizeof(int));
  if (w) {
    SAB_CHECK(cap >= (int64_t)t.w.size(), "tap capacity %lld < %zu", (long long)cap, t.w.size());
    memcpy(w, t.w.data(), t.w.size() * sizeof(float));
  }
  SAB_API_END
}

int sab_resample(sab_engine* e, const sab_resample_seg* segs, int n_segs, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(n_segs >= 0 && (segs || n_segs == 0), "bad segment list (n_segs=%d)", n_segs);
  // every rule on the host first: tables are built from integer rules alone, so the tap spans are known here
  std::vector<ResampleTable> tabs;
  std::map<std::pair<int, int>, size_t> tab_of;
  for (int i = 0; i < n_segs; ++i) {
    const sab_resample_seg& g = segs[i];
    SAB_CHECK(g.struct_bytes == (int32_t)sizeof(sab_resample_seg),
              "sab_resample_seg.struct_bytes=%d but the library's descriptor has %d bytes (header and binding differ)",
              g.struct_bytes, (int)sizeof(sab_resample_seg));
    SAB_CHECK(resample_rate_ok(g.orig_rate) && resample_rate_ok(g.new_rate),
              "segment %d: rates %d -> %d: both must lie in [8000, 192000]", i, g.orig_rate, g.new_rate);
    SAB_CHECK(g.channels >= 1 && g.channels <= 8, "segment %d: channels=%d outside 1..8", i, g.channels);
    SAB_CHECK(g.in_count >= 0 && g.out_count >= 0 && g.out_first >= 0 && g.length >= -1,
              "segment %d: negative count (in_count=%lld, out_first=%lld, out_count=%lld, length=%lld)", i,
              (long long)g.in_count, (long long)g.out_first, (long long)g.out_count, (long long)g.length);
    SAB_CHECK(g.channels == 1 || g.in_channel_stride >= g.in_count, "segment %d: channel stride %lld < in_count %lld", i,
              (long long)g.in_channel_stride, (long long)g.in_count);
    if (g.out_count == 0) continue;
    SAB_CHECK(g.out != nullptr, "segment %d: null output", i);
    const std::pair<int, int> key{g.orig_rate, g.new_rate};
    if (!tab_of.count(key)) {
      tab_of[key] = tabs.size();
      tabs.push_back(resample_table(g.orig_rate, g.new_rate));
    }
    const ResampleTable& t = tabs[tab_of[key]];
    if (g.length >= 0) {
      const int64_t n_out = ceil_div((int64_t)t.n * g.length, t.o);
      SAB_CHECK(g.out_first + g.out_count <= n_out, "segment %d: outputs [%lld, %lld) past the %lld of a %lld-sample signal",
                i, (long long)g.out_first, (long long)(g.out_first + g.out_count), (long long)n_out, (long long)g.length);
    }
    const int64_t q0 = g.out_first, q1 = g.out_first + g.out_count - 1;
    int64_t a = (q0 / t.n) * t.o + t.lo[q0 % t.n];
    int64_t b = (q1 / t.n) * t.o + t.lo[q1 % t.n] + t.K;
    a = a < 0 ? 0 : a;
    if (g.length >= 0) b = b < g.length ? b : g.length;
    if (a < b) {
      SAB_CHECK(g.in != nullptr, "segment %d: null input", i);
      SAB_CHECK(a >= g.in_first && b <= g.in_first + g.in_count,
                "segment %d: outputs [%lld, %lld) read input samples [%lld, %lld), the buffer holds [%lld, %lld)", i,
                (long long)q0, (long long)(q1 + 1), (long long)a, (long long)b, (long long)g.in_first,
                (long long)(g.in_first + g.in_count));
    }
    SAB_CHECK(g.out_count <= (int64_t)RS_BLOCK * (INT32_MAX / 2), "segment %d: %lld outputs is too many for one call", i,
              (long long)g.out_count);
  }
  SAB_CHECK(e != nullptr, "null engine");
  DeviceGuard _dg(e->device);
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<ResampleSeg> dev;
  int64_t ctas = 0, tab_floats = 0, span = 0;
  double bytes = 0;
  for (int i = 0; i < n_segs; ++i) {
    const sab_resample_seg& g = segs[i];
    if (g.out_count == 0) continue;
    const ResampleTableDev& t = resample_table_dev(e, g.orig_rate, g.new_rate);
    ResampleSeg s{g.in, g.in_channel_stride, g.in_first, g.in_count, g.length, g.out, g.out_first, g.out_count,
                  t.w, t.lo, t.o, t.n, t.K, g.channels, (int)ctas, (int64_t)t.n * t.K <= RS_SMEM_TABLE};
    dev.push_back(s);
    ctas += (g.out_count + RS_BLOCK - 1) / RS_BLOCK;
    if (s.smem_table) tab_floats = std::max<int64_t>(tab_floats, (int64_t)t.n * t.K);
    // a CTA's outputs q0 .. q0 + RS_BLOCK - 1 read m o + lo[j] within [q o / n - R, q o / n - R + 1) from the first
    // to K past the last
    span = std::max<int64_t>(span, ceil_div((int64_t)(RS_BLOCK - 1) * t.o, t.n) + t.K + 2);
    bytes += 4.0 * (double)g.out_count * (1.0 + (double)g.channels * t.o / t.n);
  }
  SAB_CHECK(ctas <= INT32_MAX, "%lld CTAs is too many for one call", (long long)ctas);
  if (dev.empty()) return 0;
  const int64_t smem = (tab_floats + span) * (int64_t)sizeof(float);
  SAB_CHECK(smem <= RS_MAX_SMEM, "resampling needs %lld B of shared memory (at most %d)", (long long)smem, RS_MAX_SMEM);
  if ((int64_t)dev.size() > e->rs_desc_cap) {
    SAB_CUDA(cudaStreamSynchronize(st));           // the old list may still be read by an earlier launch
    e->rs_desc_pool.release();
    e->rs_desc_cap = std::max<int64_t>(64, (int64_t)dev.size());
    e->rs_desc = e->rs_desc_pool.alloc<ResampleSeg>(e->rs_desc_cap);
  }
  SAB_CUDA(cudaMemcpyAsync(e->rs_desc, dev.data(), dev.size() * sizeof(ResampleSeg), cudaMemcpyHostToDevice, st));
  ensure_dynamic_smem(reinterpret_cast<const void*>(resample_kernel), RS_MAX_SMEM);
  mark(e, st, "resample", 0, bytes);
  resample_kernel<<<(unsigned)ctas, RS_THREADS, (size_t)smem, st>>>(e->rs_desc, (int)dev.size(), (int)tab_floats);
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

// ---- multichannel stems (spread_channels.cuh) ----
// The twiddles exp(-2 pi i m / N), m < N / 2, then the periodic Hann window, evaluated in float64 and rounded once.
static const float2* spread_table_dev(sab_engine* e) {
  if (!e->sp_table) {
    std::vector<float2> h(SP_N / 2 + SP_N / 2);          // N / 2 twiddles, then N window floats as N / 2 float2
    float* win = reinterpret_cast<float*>(h.data() + SP_N / 2);
    const double pi = 3.14159265358979323846;
    for (int m = 0; m < SP_N / 2; ++m)
      h[m] = make_float2((float)cos(2.0 * pi * m / SP_N), (float)-sin(2.0 * pi * m / SP_N));
    for (int n = 0; n < SP_N; ++n) win[n] = (float)(0.5 - 0.5 * cos(2.0 * pi * n / SP_N));
    float2* d = e->sp_table_pool.alloc<float2>((int64_t)h.size());
    SAB_CUDA(cudaMemcpy(d, h.data(), h.size() * sizeof(float2), cudaMemcpyHostToDevice));
    e->sp_table = d;
  }
  return e->sp_table;
}

// Does the window [first, first + count) of a signal of `length` samples (< 0: unknown) hold every index of [a, b)
// that is >= 0 and below the known length?
static bool spread_window_holds(int64_t first, int64_t count, int64_t length, int64_t a, int64_t b) {
  a = a < 0 ? 0 : a;
  if (length >= 0) b = b < length ? b : length;
  return a >= b || (a >= first && b <= first + count);
}

int sab_spread_channels(sab_engine* e, const sab_spread_seg* segs, int n_segs, void* stream) {
  SAB_API_BEGIN
  SAB_CHECK(n_segs >= 0 && (segs || n_segs == 0), "bad segment list (n_segs=%d)", n_segs);
  for (int i = 0; i < n_segs; ++i) {
    const sab_spread_seg& g = segs[i];
    SAB_CHECK(g.struct_bytes == (int32_t)sizeof(sab_spread_seg),
              "sab_spread_seg.struct_bytes=%d but the library's descriptor has %d bytes (header and binding differ)",
              g.struct_bytes, (int)sizeof(sab_spread_seg));
    SAB_CHECK(g.channels >= 1 && g.channels <= 8, "segment %d: channels=%d outside 1..8", i, g.channels);
    SAB_CHECK(g.tr_count >= 0 && g.mix_count >= 0 && g.out_count >= 0 && g.out_first >= 0 && g.tr_length >= -1 &&
                  g.mix_length >= -1,
              "segment %d: negative count (tr_count=%lld, mix_count=%lld, out_first=%lld, out_count=%lld, "
              "tr_length=%lld, mix_length=%lld)", i, (long long)g.tr_count, (long long)g.mix_count,
              (long long)g.out_first, (long long)g.out_count, (long long)g.tr_length, (long long)g.mix_length);
    SAB_CHECK(g.channels == 1 || g.mix_channel_stride >= g.mix_count, "segment %d: mix channel stride %lld < mix_count %lld",
              i, (long long)g.mix_channel_stride, (long long)g.mix_count);
    SAB_CHECK(g.channels == 1 || g.out_channel_stride >= g.out_count,
              "segment %d: output channel stride %lld < out_count %lld", i, (long long)g.out_channel_stride,
              (long long)g.out_count);
    SAB_CHECK(g.tr_length < 0 || g.mix_length < 0 || g.mix_length <= g.tr_length,
              "segment %d: a mixture of %lld samples is longer than its %lld-sample stems", i, (long long)g.mix_length,
              (long long)g.tr_length);
    if (g.out_count == 0) continue;
    SAB_CHECK(g.out_target && g.out_residual, "segment %d: null output", i);
    SAB_CHECK(g.tr_length < 0 || g.out_first + g.out_count <= g.tr_length,
              "segment %d: outputs [%lld, %lld) past the end of %lld-sample stems", i, (long long)g.out_first,
              (long long)(g.out_first + g.out_count), (long long)g.tr_length);
    // outputs [s0, s1) read the frames floor(s0 / a) .. floor((s1 - 1) / a) + 3
    const int64_t s0 = g.out_first, s1 = g.out_first + g.out_count;
    const int64_t a = (s0 / SP_HOP - 3) * SP_HOP, b = ((s1 - 1) / SP_HOP + 4) * SP_HOP;
    const int64_t bt = g.tr_length >= 0 && g.tr_length < b ? g.tr_length : b;
    const int64_t bx = g.mix_length >= 0 && g.mix_length < b ? g.mix_length : b;
    SAB_CHECK(spread_window_holds(g.tr_first, g.tr_count, g.tr_length, a, b),
              "segment %d: outputs [%lld, %lld) read stem samples [%lld, %lld), the buffers hold [%lld, %lld) (length "
              "%lld)", i, (long long)s0, (long long)s1, (long long)(a < 0 ? 0 : a), (long long)bt, (long long)g.tr_first,
              (long long)(g.tr_first + g.tr_count), (long long)g.tr_length);
    SAB_CHECK(spread_window_holds(g.mix_first, g.mix_count, g.mix_length, a, b),
              "segment %d: outputs [%lld, %lld) read mixture samples [%lld, %lld), the buffer holds [%lld, %lld) "
              "(length %lld)", i, (long long)s0, (long long)s1, (long long)(a < 0 ? 0 : a), (long long)bx,
              (long long)g.mix_first, (long long)(g.mix_first + g.mix_count), (long long)g.mix_length);
    SAB_CHECK((g.target && g.residual) || spread_window_holds(0, 0, g.tr_length, a, b), "segment %d: null stems", i);
    SAB_CHECK(g.mix || spread_window_holds(0, 0, g.mix_length, a, b), "segment %d: null mixture", i);
    SAB_CHECK(g.out_count <= (int64_t)SP_SPAN * (INT32_MAX / 2), "segment %d: %lld outputs is too many for one call", i,
              (long long)g.out_count);
  }
  SAB_CHECK(e != nullptr, "null engine");
  DeviceGuard _dg(e->device);
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<SpreadSeg> dev;
  int64_t ctas = 0;
  int c_max = 1;
  double bytes = 0;
  for (int i = 0; i < n_segs; ++i) {
    const sab_spread_seg& g = segs[i];
    if (g.out_count == 0) continue;
    SpreadSeg s{g.target, g.residual, g.tr_first, g.tr_count, g.tr_length, g.mix, g.mix_channel_stride, g.mix_first,
                g.mix_count, g.mix_length, g.out_target, g.out_residual, g.out_channel_stride, g.out_first, g.out_count,
                g.channels, (int)ctas};
    dev.push_back(s);
    const int64_t h0 = g.out_first / SP_HOP, h1 = (g.out_first + g.out_count - 1) / SP_HOP;
    ctas += (h1 - h0) / SP_HOPS + 1;
    c_max = std::max(c_max, (int)g.channels);
    bytes += 4.0 * (double)g.out_count * (2.0 + 3.0 * g.channels);
  }
  SAB_CHECK(ctas <= INT32_MAX, "%lld CTAs is too many for one call", (long long)ctas);
  if (dev.empty()) return 0;
  const float2* table = spread_table_dev(e);
  if ((int64_t)dev.size() > e->sp_desc_cap) {
    SAB_CUDA(cudaStreamSynchronize(st));           // the old list may still be read by an earlier launch
    e->sp_desc_pool.release();
    e->sp_desc_cap = std::max<int64_t>(64, (int64_t)dev.size());
    e->sp_desc = e->sp_desc_pool.alloc<SpreadSeg>(e->sp_desc_cap);
  }
  SAB_CUDA(cudaMemcpyAsync(e->sp_desc, dev.data(), dev.size() * sizeof(SpreadSeg), cudaMemcpyHostToDevice, st));
  ensure_dynamic_smem(reinterpret_cast<const void*>(spread_channels_kernel), SP_MAX_SMEM);
  const int64_t smem = SP_SMEM_FIXED + (int64_t)c_max * SP_SPAN * (int64_t)sizeof(float);
  mark(e, st, "spread_channels", 0, bytes);
  spread_channels_kernel<<<(unsigned)ctas, SP_THREADS, (size_t)smem, st>>>(e->sp_desc, (int)dev.size(), table);
  SAB_CUDA(cudaGetLastError());
  SAB_API_END
}

}  // extern "C"

#include "t5_engine.inc"
