// libdiamond_b200.so — C ABI (include/diamond_b200.h) over the sm_90a kernels.
#include <cstdlib>
#include <memory>
#include <mutex>
#include <map>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "../../include/diamond_b200.h"
#include "aux_kernels.cuh"
#include "conv_tc.cuh"
#include "wgrad_tc.cuh"
#include "bwd_kernels.cuh"
#include "optim_kernels.cuh"

using namespace dmd;

// ---------------------------------------------------------------------------------------------- errors / counters
static thread_local std::string g_err;
static thread_local long long g_launches = 0;

static int fail(const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_err = buf;
  return 1;
}
#define DMD_CHECK(cond, ...) \
  do {                       \
    if (!(cond)) return fail(__VA_ARGS__); \
  } while (0)
#define DMD_CUDA(expr)                                                                   \
  do {                                                                                   \
    cudaError_t e__ = (expr);                                                            \
    if (e__ != cudaSuccess) { (void)cudaGetLastError(); return fail("%s failed: %s", #expr, cudaGetErrorString(e__)); } \
  } while (0)
#define DMD_LAUNCH_OK()                                                                 \
  do {                                                                                  \
    ++g_launches;                                                                       \
    cudaError_t e__ = cudaGetLastError();                                               \
    if (e__ != cudaSuccess) return fail("kernel launch failed: %s (%s:%d)", cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

// the checks of a dmd_u8_frames argument, each named in its message; out: the kernels' copy
static int u8_frames_arg(const char* who, const char* name, const dmd_u8_frames* f, U8Frames* out) {
  DMD_CHECK(f, "%s: %s is NULL", who, name);
  DMD_CHECK(f->levels, "%s: %s->levels is NULL", who, name);
  DMD_CHECK(f->kinds, "%s: %s->kinds is NULL", who, name);
  DMD_CHECK(f->table, "%s: %s->table is NULL", who, name);
  DMD_CHECK(((uintptr_t)f->table & 3) == 0, "%s: %s->table is not 4-byte aligned", who, name);
  DMD_CHECK(f->batch_stride >= 0 && f->frame_stride >= 0, "%s: %s->batch_stride / frame_stride must be >= 0 (got %lld, %lld)", who,
            name, f->batch_stride, f->frame_stride);
  DMD_CHECK(f->kind_batch_stride >= 0 && f->kind_frame_stride >= 0,
            "%s: %s->kind_batch_stride / kind_frame_stride must be >= 0 (got %lld, %lld)", who, name, f->kind_batch_stride,
            f->kind_frame_stride);
  *out = U8Frames{f->levels, f->batch_stride, f->frame_stride, f->kinds, f->kind_batch_stride, f->kind_frame_stride, f->table};
  return 0;
}

extern "C" int dmd_version(void) { return DMD_VERSION; }
extern "C" const char* dmd_last_error(void) { return g_err.c_str(); }
extern "C" long long dmd_launch_count(int reset) {
  long long v = g_launches;
  if (reset) g_launches = 0;
  return v;
}

// ---- kernel trace (diagnostics; scripts/ktrace.py): launches issued between dmd_ktrace_begin and dmd_ktrace_end get one slot
// each in a device buffer and stamp the GPU nanosecond timer when their inputs are ready
static long long* g_kt_buf = nullptr;
static int g_kt_cap = 0, g_kt_n = 0;
static bool g_kt_on = false;
static std::vector<std::string> g_kt_names;
static long long* kt_slot(const char* kind, int grid, int aux) {
  if (!g_kt_on || g_kt_n >= g_kt_cap) return nullptr;
  char buf[96];
  snprintf(buf, sizeof(buf), "%s grid=%d aux=%d", kind, grid, aux);
  g_kt_names.push_back(buf);
  return g_kt_buf + g_kt_n++;
}
extern "C" int dmd_ktrace_begin(int capacity) {
  if (g_kt_cap < capacity) {
    if (g_kt_buf) cudaFree(g_kt_buf);
    if (cudaMalloc(&g_kt_buf, (size_t)capacity * 8) != cudaSuccess) { g_kt_buf = nullptr; g_kt_cap = 0; g_err = "ktrace: cudaMalloc failed"; return 1; }
    g_kt_cap = capacity;
  }
  cudaMemset(g_kt_buf, 0, (size_t)g_kt_cap * 8);
  g_kt_n = 0; g_kt_names.clear(); g_kt_on = true;
  return 0;
}
// stops assigning slots; copies the stamps (ns) to `stamps` and returns the number of traced launches (call after a device sync)
extern "C" int dmd_ktrace_end(long long* stamps, int capacity) {
  g_kt_on = false;
  const int n = g_kt_n < capacity ? g_kt_n : capacity;
  if (n > 0 && stamps) cudaMemcpy(stamps, g_kt_buf, (size_t)n * 8, cudaMemcpyDeviceToHost);
  return n;
}
extern "C" const char* dmd_ktrace_name(int i) { return (i >= 0 && i < (int)g_kt_names.size()) ? g_kt_names[i].c_str() : ""; }

static inline int round_up(int x, int m) { return (x + m - 1) / m * m; }
// SM count of the H100 SXM the launch shapes of the memory-bound kernels are planned for (grids of >= 2 blocks per SM).  A plan
// does not depend on the device it is built on, so host-only planning (dmd_prep_plan) gives the same answer as a launch.
constexpr int kPlanSms = 132;
// widest conditioning vector (cond_channels) the denoiser and reward / termination model accept: film_wgrad_kernel covers it in
// 256-column slices, and the split-K partials of dcond = dfilm Wf get their own buffer when the backward temporaries hold too few
// (make_train_plan)
constexpr int kMaxCondChannels = 2048;
static inline int gn_group_size(int C) {  // blocks.py:12,27: num_groups = max(1, C // 32)
  int G = C / 32 > 1 ? C / 32 : 1;
  return C / G;
}

// ---------------------------------------------------------------------------------------------- conv launcher
static size_t plc16_bytes(int B, int H, int W, int C) {
  const Plc g = plc_geometry(B, H, W);
  return (size_t)(round_up(C, 16) / 8) * g.Qalloc * 16;
}
extern "C" size_t dmd_plc16_bytes(int B, int H, int W, int C) { return plc16_bytes(B, H, W, C); }

// The statistics epilogue keeps kStatSlots images per 128-position tile, so the (padded) input image must hold at least 64
// positions: 7x7 and up.  The executors follow a conv on a smaller image with gn_stats instead (PlanBuilder::conv).
static bool conv_epilogue_stats_fit(int H, int W) { const Plc g = plc_geometry(1, H, W); return g.PH * g.PW >= 64; }

static int conv_fill(const dmd_conv_desc* d, ConvParams* p, size_t* smem, int* acc_cols) {
  DMD_CHECK(d->src0 && d->out && d->wpk, "conv: null src0/out/wpk");
  DMD_CHECK(d->taps == 9 || d->taps == 1, "conv: taps must be 1 or 9 (got %d)", d->taps);
  DMD_CHECK(d->stride == 1 || d->stride == 2, "conv: stride must be 1 or 2");
  DMD_CHECK(d->C0 > 0 && d->C0 % 16 == 0 && d->C1 % 16 == 0 && d->C0 + d->C1 <= kMaxCin, "conv: operand channels must be multiples of 16, total <= %d (C0=%d C1=%d)", kMaxCin, d->C0, d->C1);
  DMD_CHECK((d->C1 == 0) == (d->src1 == nullptr), "conv: src1/C1 mismatch");
  if (d->precise) DMD_CHECK(d->src0_lo && ((d->C1 == 0) == (d->src1_lo == nullptr)), "conv: precise mode needs the low operand parts");
  DMD_CHECK(d->CoutPad % 16 == 0 && d->CoutPad >= 16 && d->CoutPad <= 128 && d->Cout <= d->CoutPad && d->Cout > 0, "conv: bad Cout=%d CoutPad=%d", d->Cout, d->CoutPad);
  memset(p, 0, sizeof(*p));
  {
    const uint8_t* hi[2] = {(const uint8_t*)d->src0, (const uint8_t*)d->src1};
    const uint8_t* lo[2] = {(const uint8_t*)d->src0_lo, (const uint8_t*)d->src1_lo};
    const int cs[2] = {d->C0, d->C1};
    const int nsrc = d->C1 ? 2 : 1;
    int n = 0;
    for (int rep = 0; rep < (d->precise ? 3 : 1); ++rep)  // [hi | lo | hi] against weights [W_hi | W_hi | W_lo]
      for (int k = 0; k < nsrc; ++k) { p->seg_base[n] = (rep == 1) ? lo[k] : hi[k]; p->seg_slabs[n] = cs[k] / 16; ++n; }
    p->Cin = (d->C0 + d->C1) * (d->precise ? 3 : 1);
    p->Cextra = 0;
    if (d->wpk_x) {  // fused split-fp16 1x1 projection: [x_hi | x_lo | x_hi] against [W_hi | W_hi | W_lo], centre tap only
      DMD_CHECK(d->xsrc0 && d->xsrc0_lo && d->xC0 > 0 && d->xC0 % 16 == 0 && d->xC1 % 16 == 0 && d->xC0 + d->xC1 <= kMaxCin, "conv: bad fused projection operands");
      DMD_CHECK((d->xC1 == 0) == (d->xsrc1 == nullptr) && (d->xC1 == 0) == (d->xsrc1_lo == nullptr), "conv: fused projection src1 mismatch");
      const uint8_t* xh[2] = {(const uint8_t*)d->xsrc0, (const uint8_t*)d->xsrc1};
      const uint8_t* xl[2] = {(const uint8_t*)d->xsrc0_lo, (const uint8_t*)d->xsrc1_lo};
      const int xc[2] = {d->xC0, d->xC1};
      // the hi parts are loaded ONCE and multiplied by both W_hi and W_lo (two MMAs per slab), the lo parts by W_hi: 2/3 of the
      // slabs of the naive [x_hi | x_lo | x_hi] K order, and each slab holds only the tile's own 128 rows (centre tap: no halo)
      for (int rep = 0; rep < 2; ++rep)
        for (int k = 0; k < (d->xC1 ? 2 : 1); ++k) {
          DMD_CHECK(n < kMaxSegs, "conv: too many operand segments");
          p->seg_base[n] = (rep == 1) ? xl[k] : xh[k]; p->seg_slabs[n] = xc[k] / 16; ++n;
        }
      p->Cextra = 3 * (d->xC0 + d->xC1);
      p->xslabs = 2 * (d->xC0 + d->xC1) / 16;
      p->wpk_extra = reinterpret_cast<const __half*>(d->wpk_x);
      p->bias_extra = d->bias_x;
    }
    p->nseg = n;
  }
  p->B = d->B; p->H = d->H; p->W = d->W; p->taps = d->taps; p->stride = d->stride;
  if (d->stride == 2) DMD_CHECK(p->H % 2 == 0 && p->W % 2 == 0, "conv: stride 2 needs even H,W");
  p->wpk = reinterpret_cast<const __half*>(d->wpk); p->bias = d->bias; p->Cout = d->Cout; p->CoutPad = d->CoutPad;
  p->resid = d->residual; p->out = d->out; p->ostats = d->out_stats; p->ogs = d->out_gs > 0 ? d->out_gs : d->Cout;
  const Plc g = plc_geometry(d->B, d->H, d->W);
  p->PW = g.PW; p->PH = g.PH; p->Q = g.Q; p->G = g.G; p->plane_bytes = (unsigned long long)g.Qalloc * 16;
  DMD_CHECK((long long)g.Q * (g.PW > g.PH ? g.PW : g.PH) < (1ll << 32), "conv: problem too large for 32-bit position math");
  const int halo = d->taps == 9 ? g.PW + 1 : 0;
  p->P = kTileM + 2 * halo; p->Palloc = p->P | 1;
  if (d->out_stats) {
    const int L4 = d->Cout / 4;
    DMD_CHECK(conv_epilogue_stats_fit(d->H, d->W), "conv: image too small for the statistics epilogue (a tile may touch at most %d images)", kStatSlots);
    DMD_CHECK(d->Cout % 4 == 0 && (L4 == 4 || L4 == 8 || L4 == 16 || L4 == 32), "conv: out_stats needs Cout in {16,32,64,128} (got %d)", d->Cout);
    DMD_CHECK(d->out_gs == 16 || d->out_gs == 32 || d->out_gs == 64 || d->out_gs == 128, "conv: out_gs must be 16/32/64/128");
    DMD_CHECK(d->Cout % d->out_gs == 0 && d->Cout / d->out_gs <= kMaxOutGroups, "conv: bad output groups");
  }
  p->dPW.init(g.PW); p->dPH.init(g.PH);
  p->num_tiles = (g.Q + kTileM - 1) / kTileM;
  // slab ring: everything that fits next to the resident weights (227 KB of shared memory per block), at most four tiles' worth
  const int kslabs = p->Cin / 16 + p->xslabs;
  const uint32_t w_bytes = conv_weight_bytes(p->taps, p->Cin, p->Cextra, p->CoutPad);
  const ConvSmemLayout L0 = conv_smem_layout(w_bytes, p->Palloc, 0);
  const long long budget = 227ll * 1024 - (long long)L0.total;
  int stages = budget > 0 ? (int)(budget / (long long)L0.slab_bytes) : 0;
  if (stages > 4 * kslabs) stages = 4 * kslabs;
  if (stages > kMaxStages) stages = kMaxStages;
  DMD_CHECK(stages >= 2, "conv: shared memory too small for W=%d Cin=%d CoutPad=%d", p->W, p->Cin, p->CoutPad);
  p->stages = stages;
  *smem = conv_smem_layout(w_bytes, p->Palloc, stages).total;
  *acc_cols = d->CoutPad <= 16 ? 16 : (d->CoutPad <= 32 ? 32 : (d->CoutPad <= 64 ? 64 : 128));   // wgmma N: a power of two
  return 0;
}

// Per-device state: SM count, the >48 KB dynamic shared memory opt-ins (function attributes are per device) and a small
// all-zero buffer (source of the zero row groups of the wgrad kernel).  Initialised on first use of each device, never
// during stream capture.
struct DevState { int num_sms = 0; void* zeros = nullptr; };
static thread_local int g_num_sms = 0;
static thread_local const uint8_t* g_zeros = nullptr;
static int init_kernels() {
  static std::mutex mu;
  static std::map<int, DevState> states;
  int dev = 0;
  DMD_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(mu);
  auto it = states.find(dev);
  if (it == states.end()) {
    DevState st;
    DMD_CUDA(cudaDeviceGetAttribute(&st.num_sms, cudaDevAttrMultiProcessorCount, dev));
    DMD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<16, 9>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<32, 9>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<64, 9>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<128, 9>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<16, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<32, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(conv_tc_kernel<128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(wgrad_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(attn_cluster_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(attn_cluster_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(attn_cluster_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, 168 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<64, kAttnL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<32, kAttnL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<64, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(attn_bwd_kernel<32, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(linear_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(linear_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    DMD_CUDA(cudaFuncSetAttribute(linear_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    DMD_CUDA(cudaMalloc(&st.zeros, 4096));
    DMD_CUDA(cudaMemset(st.zeros, 0, 4096));
    it = states.emplace(dev, st).first;
  }
  g_num_sms = it->second.num_sms;
  g_zeros = (const uint8_t*)it->second.zeros;
  return 0;
}

// Launch with programmatic stream serialization: the kernel may become resident while its predecessor drains and runs
// its prologue up to griddepcontrol.wait.  Captured into CUDA graphs as a programmatic dependency edge.
template <typename Kernel, typename Params>
static int launch_pdl(Kernel kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t st, const Params& p) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  DMD_CUDA(cudaLaunchKernelEx(&cfg, kernel, p));
  DMD_LAUNCH_OK();
  return 0;
}

template <int kCols>
static int conv_launch_t(const ConvParams& p0, size_t smem, cudaStream_t st) {
  if (init_kernels()) return 1;
  const int grid = p0.num_tiles < g_num_sms ? p0.num_tiles : g_num_sms;  // persistent: one CTA per SM
  ConvParams p = p0;
  p.ktrace = kt_slot(p.taps == 9 ? "conv3x3" : "conv1x1", p.num_tiles, (p.Cin + p.Cextra) * 1000 + p.W);
  if (p.taps == 9) return launch_pdl(conv_tc_kernel<kCols, 9>, dim3(grid), dim3(kConvThreads), smem, st, p);
  return launch_pdl(conv_tc_kernel<kCols, 1>, dim3(grid), dim3(kConvThreads), smem, st, p);
}

// ---- prep (GroupNorm / AdaGroupNorm / SiLU / upsample -> PLC16 operand)
static int prep_fill(const dmd_prep_desc* d, PrepParams* p, int* nsrc) {
  DMD_CHECK(d->src0 && d->dst0, "prep: null src0/dst0");
  DMD_CHECK(d->C0 % 8 == 0 && d->C1 % 8 == 0 && d->C0 > 0 && d->C0 <= kMaxCin && d->C1 <= kMaxCin, "prep: channels must be multiples of 8 (C0=%d C1=%d)", d->C0, d->C1);
  DMD_CHECK((d->C1 == 0) == (d->src1 == nullptr) && (d->C1 == 0) == (d->dst1 == nullptr), "prep: src1/dst1/C1 mismatch");
  DMD_CHECK(d->mode >= 0 && d->mode <= 2, "prep: bad mode");
  for (int c : {d->C0, d->C1 ? d->C1 : 16}) {
    const int cp = round_up(c, 16);
    DMD_CHECK(cp == 16 || cp == 32 || cp == 64 || cp == 128, "prep: a source must have <= 16/32/64/128 channels after padding (got %d)", c);
  }
  memset(p, 0, sizeof(*p));
  p->s[0].src = d->src0; p->s[0].C = d->C0; p->s[0].Cpad = round_up(d->C0, 16); p->s[0].stats = d->stats0; p->s[0].gs = d->gs0 > 0 ? d->gs0 : 8;
  p->s[0].c_offset = 0; p->s[0].dst = (uint8_t*)d->dst0; p->s[0].dst_raw = (uint8_t*)d->dst_raw0;
  p->s[0].dst_lo = (uint8_t*)d->dst_lo0; p->s[0].dst_raw_lo = (uint8_t*)d->dst_raw_lo0;
  p->s[1].dst_lo = (uint8_t*)d->dst_lo1; p->s[1].dst_raw_lo = (uint8_t*)d->dst_raw_lo1;
  DMD_CHECK(!(d->dst_raw_lo0 && !d->dst_raw0) && !(d->dst_raw_lo1 && !d->dst_raw1), "prep: raw low part needs the raw operand too");
  p->s[1].src = d->src1; p->s[1].C = d->C1; p->s[1].Cpad = round_up(d->C1 > 0 ? d->C1 : 16, 16); p->s[1].stats = d->stats1; p->s[1].gs = d->gs1 > 0 ? d->gs1 : 8;
  p->s[1].c_offset = d->C0; p->s[1].dst = (uint8_t*)d->dst1; p->s[1].dst_raw = (uint8_t*)d->dst_raw1;
  if (d->mode) {
    DMD_CHECK(d->stats0 && d->gs0 > 0 && d->C0 % d->gs0 == 0, "prep: norm mode needs stats0/gs0");
    if (d->C1) DMD_CHECK(d->stats1 && d->gs1 > 0 && d->C1 % d->gs1 == 0, "prep: norm mode needs stats1/gs1");
    if (d->mode == 1) DMD_CHECK(d->film != nullptr, "prep: AdaGroupNorm needs film");
    if (d->mode == 2) DMD_CHECK(d->gamma && d->beta, "prep: GroupNorm needs gamma/beta");
    DMD_CHECK(d->upsample == 0, "prep: norm + upsample unsupported");
  }
  p->B = d->B; p->Hs = d->Hs; p->Ws = d->Ws; p->ups = d->upsample;   // 1 nearest-2x, 2 zero insertion (stride-2 adjoint)
  DMD_CHECK(d->upsample >= 0 && d->upsample <= 2, "prep: upsample must be 0, 1 (nearest 2x) or 2 (zero insertion)");
  DMD_CHECK(d->upsample != 2 || (d->mode == 0 && !d->silu && d->C1 == 0 && !d->dst_raw0 && !d->dst_lo0), "prep: zero insertion is a raw single-source operand");
  p->H = d->upsample ? 2 * d->Hs : d->Hs; p->W = d->upsample ? 2 * d->Ws : d->Ws;
  p->mode = d->mode; p->act = d->silu ? 1 : 0;
  p->film = d->film; p->film_stride = d->film_stride; p->film_off = d->film_off; p->film_ctot = d->C0 + d->C1;
  p->gamma = d->gamma; p->beta = d->beta; p->eps = d->eps;
  const Plc g = plc_geometry(d->B, p->H, p->W);
  // 4x4 (25 padded positions) is the smallest image the executors build
  DMD_CHECK(g.PH * g.PW >= 25, "prep: image too small (%dx%d; 4x4 is the smallest)", p->H, p->W);
  // a block touches at most 2 images (at most PH * PW positions); low-resolution levels get smaller blocks so that the grid
  // still covers the SMs.  Multiples of 32 positions, 16 on images of fewer than 32 (4x4, 4x5)
  int ppb = g.PH * g.PW >= 256 ? 256 : (g.PH * g.PW / 32) * 32;
  while (ppb > 64 && (g.Qalloc + ppb - 1) / ppb < 2 * kPlanSms) ppb >>= 1;
  ppb = (ppb / 32) * 32;
  if (ppb == 0) ppb = 16;
  p->pos_per_block = ppb;
  // both kernels keep (mean, rstd) of at most 4 groups per image slot in shared memory, for every source
  DMD_CHECK(d->mode == 0 || (d->C0 / (d->gs0 > 0 ? d->gs0 : 8) <= 4 && d->C1 / (d->gs1 > 0 ? d->gs1 : 8) <= 4),
            "prep: at most 4 groups per source (C0=%d gs0=%d, C1=%d gs1=%d)", d->C0, d->gs0, d->C1, d->gs1);
  DMD_CHECK((long long)g.Q * (g.PW > g.PH ? g.PW : g.PH) < (1ll << 32), "prep: problem too large for 32-bit position math");
  p->PW = g.PW; p->PH = g.PH; p->Q = g.Q; p->G = g.G; p->Qalloc = g.Qalloc; p->plane_bytes = (unsigned long long)g.Qalloc * 16;
  p->dPW.init(g.PW); p->dPH.init(g.PH);
  *nsrc = d->C1 ? 2 : 1;
  return 0;
}
static int prep_launch(const PrepParams& p0, int nsrc, cudaStream_t st) {
  PrepParams p = p0;
  p.ktrace = kt_slot("prep", (p.Qalloc + p.pos_per_block - 1) / p.pos_per_block * nsrc, p.mode * 1000 + p.W);
  if (p.ups == 2) {  // zero insertion: its own kernel (single source, raw mode)
    const long long total = (long long)p.Qalloc * (p.s[0].Cpad >> 3);
    return launch_pdl(zero_insert_prep_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, st, p);
  }
  const dim3 grid((p.Qalloc + p.pos_per_block - 1) / p.pos_per_block, 1, nsrc);
  // the hot cases (norm + SiLU, no upsample, no low part of the normalised operand; raw + raw-low on every source or on none)
  // run on the lean kernel; everything else on the generic one
  bool fast = p.mode != 0 && p.act && p.ups == 0;
  const bool raw = p.s[0].dst_raw != nullptr;
  for (int k = 0; k < nsrc && fast; ++k) {
    const PrepSrc& S = p.s[k];
    if (S.dst_lo != nullptr || (S.dst_raw != nullptr) != raw || (S.dst_raw_lo != nullptr) != raw || S.Cpad != p.s[0].Cpad || S.C % 8 != 0) fast = false;
  }
  if (fast && (long long)p.B * p.Hs * p.Ws * (p.s[0].C > p.s[nsrc - 1].C ? p.s[0].C : p.s[nsrc - 1].C) >= (1ll << 31)) fast = false;   // 32-bit source indices
  if (fast) {
    const int nch = p.s[0].Cpad >> 3;
    if (nch == 8) return raw ? launch_pdl(prep_fast_kernel<8, true>, grid, dim3(kPrepThreads), 0, st, p) : launch_pdl(prep_fast_kernel<8, false>, grid, dim3(kPrepThreads), 0, st, p);
    if (nch == 4) return raw ? launch_pdl(prep_fast_kernel<4, true>, grid, dim3(kPrepThreads), 0, st, p) : launch_pdl(prep_fast_kernel<4, false>, grid, dim3(kPrepThreads), 0, st, p);
  }
  return launch_pdl(prep_act_kernel, grid, dim3(kPrepThreads), 0, st, p);
}
extern "C" int dmd_prep_plan(const dmd_prep_desc* d, int* blocks, int* pos_per_block, int* sources) {
  DMD_CHECK(d && blocks && pos_per_block && sources, "prep_plan: null argument");
  PrepParams p; int nsrc;
  if (prep_fill(d, &p, &nsrc)) return 1;
  *blocks = (p.Qalloc + p.pos_per_block - 1) / p.pos_per_block; *pos_per_block = p.pos_per_block; *sources = nsrc;
  return 0;
}
extern "C" int dmd_conv_plan(const dmd_conv_desc* d, dmd_conv_plan_info* out) {
  DMD_CHECK(d && out, "conv_plan: null argument");
  ConvParams p; size_t smem; int cols;
  if (conv_fill(d, &p, &smem, &cols)) return 1;
  out->tiles = p.num_tiles; out->kslabs = p.Cin / 16 + p.xslabs; out->stages = p.stages; out->acc_cols = cols;
  out->smem_bytes = smem; out->weight_bytes = conv_weight_bytes(p.taps, p.Cin, p.Cextra, p.CoutPad);
  return 0;
}
extern "C" int dmd_prep_act(const dmd_prep_desc* d, void* stream) {
  PrepParams p; int nsrc;
  if (prep_fill(d, &p, &nsrc)) return 1;
  return prep_launch(p, nsrc, (cudaStream_t)stream);
}

static int conv_launch(const ConvParams& p, size_t smem, int acc_cols, cudaStream_t st) {
  switch (acc_cols) {
    case 16: return conv_launch_t<16>(p, smem, st);
    case 32: return conv_launch_t<32>(p, smem, st);
    case 64: return conv_launch_t<64>(p, smem, st);
    default: return conv_launch_t<128>(p, smem, st);
  }
}

extern "C" int dmd_conv2d_fprop(const dmd_conv_desc* d, void* stream) {
  ConvParams p; size_t smem; int cols;
  if (conv_fill(d, &p, &smem, &cols)) return 1;
  return conv_launch(p, smem, cols, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------- wgrad launcher
// Fills the wgmma weight-gradient launch for one (gradient operand, activation operand) pair.  grad: PLC16, Cg stored
// channels (<= 64); act: PLC16, Ca stored channels (16 / 32 / 64), both over B images of H x W (conv INPUT size; a
// stride-2 conv passes its zero-inserted gradient).  Like conv_fill, it touches no device: the device's part of the launch (its
// SM count and zero buffer) is added by wgrad_launch.
struct WgradLaunch { WgradParams wp; WgradReduceParams rp; size_t smem; };
static size_t wgrad_partial_bytes(int num_sms) { return (size_t)num_sms * kWgTaps * 64 * 64 * sizeof(float); }

static int wgrad_fill(const void* grad, int Cg, const void* act, int Ca, int B, int H, int W, int taps, float* partial,
                      int Cout, int Cin, int CinTot, int ci_off, const float* inv_scale, int accumulate, WgradLaunch* L, int co_off = 0) {
  DMD_CHECK(grad && act && partial, "wgrad: null operand / partial buffer");
  DMD_CHECK(taps == 9 || taps == 1, "wgrad: taps must be 1 or 9");
  DMD_CHECK(Cg % 8 == 0 && Cg > 0 && Cg <= 64, "wgrad: gradient operand channels must be a multiple of 8, <= 64 (got %d)", Cg);
  DMD_CHECK(Ca == 16 || Ca == 32 || Ca == 64, "wgrad: activation operand channels must be 16, 32 or 64 (got %d)", Ca);
  DMD_CHECK(Cout > 0 && Cout <= Cg && Cin > 0 && Cin <= Ca && ci_off >= 0 && ci_off + Cin <= CinTot, "wgrad: bad channel counts");
  memset(L, 0, sizeof(*L));
  const Plc g = plc_geometry(B, H, W);
  const size_t plane = (size_t)g.Qalloc * 16;
  WgradParams& wp = L->wp;
  const int ng = Cg / 8;
  for (int j = 0; j < 8; ++j) wp.a_plane[j] = j < ng ? (const uint8_t*)grad + (size_t)j * plane : nullptr;
  wp.nB = Ca / 8;
  for (int j = 0; j < wp.nB; ++j) wp.b_plane[j] = (const uint8_t*)act + (size_t)j * plane;
  wp.taps = taps; wp.PW = g.PW; wp.halo = taps == 9 ? g.PW + 1 : 0;
  wp.G = g.G; wp.num_tiles = (g.Q + kTileM - 1) / kTileM; wp.Pb = kTileM + 2 * wp.halo;
  const WgradSmem one = wgrad_smem(wp.nB, wp.halo, 1);
  int stages = (int)((227ll * 1024 - 256) / (long long)(one.a_bytes + one.b_bytes));
  if (stages > kWgStagesMax) stages = kWgStagesMax;
  DMD_CHECK(stages >= 2, "wgrad: image too wide for the shared-memory stage (W=%d)", W);
  wp.stages = stages;
  wp.partial = partial;
  L->smem = wgrad_smem(wp.nB, wp.halo, stages).total;
  WgradReduceParams& rp = L->rp;
  rp.partial = partial; rp.N = Ca;
  rp.Cout = Cout; rp.Cin = Cin; rp.CinTot = CinTot; rp.ci_off = ci_off; rp.co_off = co_off; rp.taps = taps;
  rp.inv_scale = inv_scale; rp.accumulate = accumulate;
  return 0;
}
static int wgrad_launch(const WgradLaunch& L, float* dW, cudaStream_t st) {
  if (init_kernels()) return 1;
  WgradParams wp = L.wp;
  wp.zeros = g_zeros;
  const int grid = wp.num_tiles < g_num_sms ? wp.num_tiles : g_num_sms;   // persistent: one CTA per SM, one partial each
  const int N = wp.nB * 8;
  if (N == 16) { if (launch_pdl(wgrad_tc_kernel<16>, dim3(grid), dim3(kWgThreads), L.smem, st, wp)) return 1; }
  else if (N == 32) { if (launch_pdl(wgrad_tc_kernel<32>, dim3(grid), dim3(kWgThreads), L.smem, st, wp)) return 1; }
  else if (launch_pdl(wgrad_tc_kernel<64>, dim3(grid), dim3(kWgThreads), L.smem, st, wp)) return 1;
  WgradReduceParams rp = L.rp;
  rp.nparts = grid; rp.dW = dW;
  const int total = rp.taps * 64 * rp.N;
  wgrad_reduce_kernel<<<(total + 63) / 64, 256, 0, st>>>(rp);
  DMD_LAUNCH_OK();
  return 0;
}

extern "C" size_t dmd_wgrad_partial_bytes(void) {
  if (init_kernels()) return 0;
  return wgrad_partial_bytes(g_num_sms);
}
extern "C" int dmd_conv2d_wgrad(const dmd_wgrad_desc* d, void* stream) {
  DMD_CHECK(d && d->dW, "wgrad: null descriptor / dW");
  if (init_kernels()) return 1;
  DMD_CHECK(d->partial_bytes >= wgrad_partial_bytes(g_num_sms), "wgrad: partial buffer too small (%zu < %zu)", d->partial_bytes, wgrad_partial_bytes(g_num_sms));
  WgradLaunch L;
  if (wgrad_fill(d->grad, d->Cg, d->act, d->Ca, d->B, d->H, d->W, d->taps, (float*)d->partial, d->Cout, d->Cin, d->CinTot, d->ci_off,
                 d->inv_scale, d->accumulate, &L)) return 1;
  return wgrad_launch(L, d->dW, (cudaStream_t)stream);
}
extern "C" int dmd_pack_conv_weight_dgrad(const float* w, void* wpk, int CoutF, int CinTotF, int ci_off, int CinK, int taps, void* stream) {
  DMD_CHECK(w && wpk, "pack_T: null pointer");
  const int CinP = round_up(CoutF, 16), CoutP = round_up(CinK, 16);
  const int total = taps * CinP * CoutP;
  pack_conv_weight_T_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, (__half*)wpk, CoutF, CinTotF, ci_off, CinK, CinP, CoutP, taps);
  DMD_LAUNCH_OK();
  return 0;
}

extern "C" int dmd_pack_conv_weight(const float* w, void* wpk, int Cout, int CoutPad, int CinReal, int Cin, int taps,
                                    int c0_real, int c0_store, int precise, void* stream) {
  DMD_CHECK(w && wpk, "pack: null pointer");
  DMD_CHECK(precise >= 0 && precise <= 2, "pack: precise must be 0, 1 (split [W_hi | W_hi | W_lo]) or 2 (low parts only)");
  const int total = taps * Cin * CoutPad * (precise == 1 ? 3 : 1);
  pack_conv_weight_kernel<<<(total + 255) / 256, 256, 0, (cudaStream_t)stream>>>(w, (__half*)wpk, Cout, CoutPad, CinReal, Cin, taps, c0_real, c0_store, precise);
  DMD_LAUNCH_OK();
  return 0;
}

// GroupNorm sums of an NHWC tensor, added to stats[B][C / gs][2].  det (torch.use_deterministic_algorithms): one cluster of
// kGnDetSplit CTAs owns each (image, group) and sums it in a fixed order, in place of the fp64 atomics of up to 64 blocks per image
static int gn_stats_launch(const float* x, double* stats, int B, int HW, int C, int gs, bool det, cudaStream_t st) {
  DMD_CHECK(x && stats && gs > 0 && C % gs == 0, "gn_stats: bad arguments");
  if (det) {
    DMD_CHECK(B <= 65535 && (long long)kGnDetSplit * (C / gs) < (1ll << 31), "gn_stats: B=%d or %d groups out of range", B, C / gs);
    DMD_CHECK(C % 4 == 0 && gs % 4 == 0, "gn_stats: deterministic sums need C and gs multiples of 4 (C=%d gs=%d)", C, gs);
    gn_stats_det_kernel<<<dim3(kGnDetSplit * (C / gs), B), kGnDetThreads, 0, st>>>(x, stats, HW, C, gs);
    DMD_LAUNCH_OK();
    return 0;
  }
  long long per = (long long)HW * C;
  int chunks = (int)((per + 256 * 64 - 1) / (256 * 64));
  if (chunks < 1) chunks = 1;
  if (chunks > 64) chunks = 64;
  gn_stats_kernel<<<dim3(chunks, B), 256, 0, st>>>(x, stats, HW, C, gs);
  DMD_LAUNCH_OK();
  return 0;
}
extern "C" int dmd_gn_stats(const float* x, double* stats, int B, int HW, int C, int gs, void* stream) {
  return gn_stats_launch(x, stats, B, HW, C, gs, false, (cudaStream_t)stream);
}
extern "C" int dmd_gn_stats_det(const float* x, double* stats, int B, int HW, int C, int gs, void* stream) {
  DMD_CHECK(B > 0 && HW > 0 && C > 0, "gn_stats_det: bad arguments");
  return gn_stats_launch(x, stats, B, HW, C, gs, true, (cudaStream_t)stream);
}

// scratch of the any-L attention path (q, k, v of every token); L = 64 runs in one launch without scratch
static size_t attn_scratch_bytes(int B, int L, int C) { return L == kAttnL ? 0 : (size_t)B * L * 3 * C * sizeof(float); }

// L = 64 (the 8x8 level of a 64x64 frame): one launch of attn_cluster_kernel.  Any other L: attn_qkv_kernel, then
// attn_stream_kernel, through p.scratch (attn_scratch_bytes)
static int attn_launch(const AttnParams& p, int B, cudaStream_t st) {
  // the kernels keep (mean, rstd) of at most 8 groups
  DMD_CHECK((p.C == 128 || p.C == 64 || p.C == 32) && p.L >= 1 && p.C % p.gs == 0 && p.gs % 8 == 0 && p.C / p.gs <= 8,
            "attn: unsupported shape L=%d C=%d gs=%d (C in {32, 64, 128}, at most 8 groups of a multiple of 8 channels)", p.L, p.C, p.gs);
  // attn_cluster_kernel adds the output statistics of each CTA's C/4 channels to one GroupNorm group
  DMD_CHECK(p.L != kAttnL || p.gs % (p.C / 4) == 0, "attn: L=%d needs gs a multiple of C/4 (C=%d gs=%d)", kAttnL, p.C, p.gs);
  if (init_kernels()) return 1;
  if (p.L != kAttnL) {
    DMD_CHECK(p.scratch && ((uintptr_t)p.scratch & 15) == 0, "attn: L=%d needs 16-byte aligned scratch of dmd_attn_scratch_bytes", p.L);
    DMD_CHECK(B >= 1 && B <= 65535, "attn: B=%d out of range", B);
    const dim3 grid((p.L + kAttnTile - 1) / kAttnTile, B);
    AttnParams pa = p;
    pa.ktrace = kt_slot("attn qkv", (int)(grid.x * grid.y), p.L);
    if (p.C == 128) attn_qkv_kernel<128><<<grid, kAttnQkvThreads, 0, st>>>(pa);
    else if (p.C == 64) attn_qkv_kernel<64><<<grid, kAttnQkvThreads, 0, st>>>(pa);
    else attn_qkv_kernel<32><<<grid, kAttnQkvThreads, 0, st>>>(pa);
    DMD_LAUNCH_OK();
    pa.ktrace = kt_slot("attn softmax", (int)(grid.x * grid.y), p.L);
    if (p.C == 128) attn_stream_kernel<128><<<grid, kAttnSThreads, 0, st>>>(pa);
    else if (p.C == 64) attn_stream_kernel<64><<<grid, kAttnSThreads, 0, st>>>(pa);
    else attn_stream_kernel<32><<<grid, kAttnSThreads, 0, st>>>(pa);
    DMD_LAUNCH_OK();
    return 0;
  }
  AttnParams pt = p;
  pt.ktrace = kt_slot("attn", B, p.C);
  // four CTAs per image (thread-block cluster), distributed shared memory for the head outputs
  const int CH = p.C / 4;
  const size_t csmem = sizeof(float) * ((size_t)p.L * (p.C + 1) * 2 + (size_t)p.L * (3 * CH + 4) + (size_t)p.L * CH + (size_t)4 * CH * p.C);
  if (p.C == 128) attn_cluster_kernel<128><<<4 * B, kAttnCThreads, csmem, st>>>(pt);   // 162 KB
  else if (p.C == 64) attn_cluster_kernel<64><<<4 * B, kAttnCThreads, csmem, st>>>(pt);
  else attn_cluster_kernel<32><<<4 * B, kAttnCThreads, csmem, st>>>(pt);
  DMD_LAUNCH_OK();
  return 0;
}

static int linear_launch(const float* in, const float* W, const float* bias, float* out, int B, int K, int F, int silu, cudaStream_t st,
                         int accumulate = 0, int hw_perm = 0) {
  DMD_CHECK(K % 4 == 0, "linear: K=%d must be a multiple of 4", K);
  DMD_CHECK(hw_perm == 0 || K % hw_perm == 0, "linear: bad hw_perm");
  if (init_kernels()) return 1;
  // enough blocks to cover the SMs: 8, 16 or 32 output features per block
  const int by = (B + 31) / 32;
  if ((long long)((F + 31) / 32) * by >= 2 * kPlanSms)
    linear_kernel<4><<<dim3((F + 31) / 32, by), 256, (size_t)(32 + 32) * kLinChunk * sizeof(float), st>>>(in, W, bias, out, B, K, F, silu, accumulate, hw_perm);
  else if ((long long)((F + 15) / 16) * by >= kPlanSms)
    linear_kernel<2><<<dim3((F + 15) / 16, by), 256, (size_t)(16 + 32) * kLinChunk * sizeof(float), st>>>(in, W, bias, out, B, K, F, silu, accumulate, hw_perm);
  else
    linear_kernel<1><<<dim3((F + 7) / 8, by), 256, (size_t)(8 + 32) * kLinChunk * sizeof(float), st>>>(in, W, bias, out, B, K, F, silu, accumulate, hw_perm);
  DMD_LAUNCH_OK();
  return 0;
}

// MaxPool2d(2) + GroupNorm partial sums of the pooled tensor; H, W: the pre-pool size, pooled to H/2 x W/2 with floor
// division like nn.MaxPool2d (an odd last row / column is in no window).  The statistics are reduced over aligned
// segments of min(gs, 32) lanes, i.e. consecutive channels of one pixel: a segment stays inside one group when gs is a power
// of two <= 32 or a multiple of 32, and warps start on a group boundary when C % 32 == 0 or 256 % C == 0.
static int maxpool2_stats_launch(const float* x, float* y, double* stats, int B, int H, int W, int C, int gs, cudaStream_t st) {
  DMD_CHECK(H >= 2 && W >= 2, "maxpool2_stats: H=%d, W=%d must be at least 2", H, W);
  DMD_CHECK((long long)(H / 2) * (W / 2) * C < (1ll << 31), "maxpool2_stats: image too large for 32-bit indices");
  if (stats) DMD_CHECK(gs > 0 && C % gs == 0 && (gs % 32 == 0 || (gs <= 32 && (gs & (gs - 1)) == 0)) && (C % 32 == 0 || 256 % C == 0),
                       "maxpool2_stats: statistics need gs a power of two <= 32 or a multiple of 32, and C %% 32 == 0 or 256 %% C == 0 (C=%d gs=%d)", C, gs);
  const int total = (H / 2) * (W / 2) * C;
  maxpool2_stats_kernel<<<dim3((total + 255) / 256, B), 256, 0, st>>>(x, y, stats, H, W, C, gs);
  DMD_LAUNCH_OK();
  return 0;
}

// LSTMCell pointwise part: gates [B][4Hd] (pre-activations, gate order i, f, g, o) and c_in -> h_out, c_out (c_out may be c_in)
static int lstm_gates_launch(const float* gates, const float* c_in, float* h_out, float* c_out, int B, int Hd, cudaStream_t st) {
  lstm_gates_kernel<<<(B * Hd + 255) / 256, 256, 0, st>>>(gates, c_in, h_out, c_out, B, Hd);
  DMD_LAUNCH_OK();
  return 0;
}

// ---- per-op entry points of the forward CUDA-core kernels (include/diamond_b200.h): validate, then the launchers the executors use
extern "C" int dmd_linear(const float* in, const float* W, const float* bias, float* out, int B, int K, int F, int silu, int accumulate,
                          int hw_perm, void* stream) {
  DMD_CHECK(in && W && out && B > 0 && K > 0 && F > 0 && hw_perm >= 0, "linear: bad arguments");
  return linear_launch(in, W, bias, out, B, K, F, silu, (cudaStream_t)stream, accumulate, hw_perm);
}
extern "C" int dmd_maxpool2_stats(const float* x, float* y, double* stats, int B, int H, int W, int C, int gs, void* stream) {
  DMD_CHECK(x && y && B > 0 && H > 0 && W > 0 && C > 0, "maxpool2_stats: bad arguments");
  DMD_CHECK(H % 2 == 0 && W % 2 == 0, "maxpool2_stats: H=%d, W=%d must be even", H, W);
  return maxpool2_stats_launch(x, y, stats, B, H, W, C, gs, (cudaStream_t)stream);
}
extern "C" int dmd_lstm_gates(const float* gates, const float* c_in, float* h_out, float* c_out, int B, int Hd, void* stream) {
  DMD_CHECK(gates && c_in && h_out && c_out && B > 0 && Hd > 0, "lstm_gates: bad arguments");
  DMD_CHECK((long long)B * Hd <= (1ll << 30), "lstm_gates: too many cells for 32-bit indices");
  return lstm_gates_launch(gates, c_in, h_out, c_out, B, Hd, (cudaStream_t)stream);
}

extern "C" int dmd_attn_fwd(const float* x, const double* stats_in, const float* gamma, const float* beta,
                            const float* wqkv, const float* bqkv, const float* wout, const float* bout, float* out,
                            double* out_stats, int B, int L, int C, int gs, float eps, void* stream) {
  AttnParams p{x, stats_in, gamma, beta, wqkv, bqkv, wout, bout, out, out_stats, L, C, gs, eps};
  return attn_launch(p, B, (cudaStream_t)stream);
}
extern "C" size_t dmd_attn_scratch_bytes(int B, int L, int C) { return B > 0 && L > 0 && C > 0 ? attn_scratch_bytes(B, L, C) : 0; }
extern "C" int dmd_attn_fwd_scratch(const float* x, const double* stats_in, const float* gamma, const float* beta,
                                    const float* wqkv, const float* bqkv, const float* wout, const float* bout, float* out,
                                    double* out_stats, int B, int L, int C, int gs, float eps, void* scratch, size_t scratch_bytes,
                                    void* stream) {
  DMD_CHECK(x && stats_in && gamma && beta && wqkv && bqkv && wout && bout && out && B > 0 && L > 0 && C > 0 && gs > 0,
            "attn_fwd_scratch: bad arguments");
  DMD_CHECK(scratch_bytes >= attn_scratch_bytes(B, L, C), "attn_fwd_scratch: scratch too small (%zu < %zu)", scratch_bytes,
            attn_scratch_bytes(B, L, C));
  AttnParams p{x, stats_in, gamma, beta, wqkv, bqkv, wout, bout, out, out_stats, L, C, gs, eps};
  p.scratch = (float*)scratch;
  return attn_launch(p, B, (cudaStream_t)stream);
}

extern "C" int dmd_nchw_to_nhwc(const float* in, float* out, int B, int C, int CP, int HW, void* stream) {
  nchw_to_nhwc_kernel<<<dim3((HW + 255) / 256, B), 256, 0, (cudaStream_t)stream>>>(in, out, C, CP, HW);
  DMD_LAUNCH_OK();
  return 0;
}
extern "C" int dmd_nhwc_to_nchw(const float* in, float* out, int B, int C, int CP, int HW, void* stream) {
  nhwc_to_nchw_kernel<<<dim3((HW + 255) / 256, B), 256, 0, (cudaStream_t)stream>>>(in, out, C, CP, HW);
  DMD_LAUNCH_OK();
  return 0;
}

// ---------------------------------------------------------------------------------------------- backward launchers
// The launch geometry of every CUDA-core backward kernel (bwd_kernels.cuh).  The denoiser and actor-critic executors and the
// per-op entry points (dmd_norm_bwd, dmd_colsum, ...) all launch through these, so the per-op tests run the executors' shapes.

// loss scale S = scale[0] from max|g| (amax_bits zeroed by the caller), 1/S in scale[1]
static int loss_scale_launch(const float* g, long long n, unsigned int* amax_bits, float* scale, cudaStream_t st) {
  absmax_kernel<<<(int)std::min<long long>(std::max<long long>((n + 255) / 256, 1), 1184), 256, 0, st>>>(g, amax_bits, n);
  DMD_LAUNCH_OK();
  loss_scale_kernel<<<1, 1, 0, st>>>(amax_bits, scale);
  DMD_LAUNCH_OK();
  return 0;
}

// column sums: up to 592 blocks of 256 / (Cb / 4) row lanes, at least 8 rows per lane.  part (deterministic mode): each block
// stores its sums to part[block][C] (part_bytes of room) and colsum_reduce_kernel adds them in block order, in place of the
// atomics.  The block count depends on rows and C only, so the order does too.
static long long colsum_blocks(long long rows, int C) {
  const int L4 = (C < 256 ? C : 256) >> 2, lanes = 256 / L4;
  const long long blocks = (rows + (long long)lanes * 8 - 1) / ((long long)lanes * 8);
  return blocks > 592 ? 592 : (blocks < 1 ? 1 : blocks);
}
static size_t colsum_partial_bytes(long long rows, int C) { return (size_t)colsum_blocks(rows, C) * C * sizeof(float); }
static int colsum_launch(const float* x, float* out, float* out2, const float* inv, long long rows, int C, int Creal, cudaStream_t st,
                         float* part = nullptr, size_t part_bytes = 0) {
  const long long blocks = colsum_blocks(rows, C);
  if (part) {
    DMD_CHECK(colsum_partial_bytes(rows, C) <= part_bytes, "colsum: partials (%lld x %d floats) exceed the partial buffer", blocks, C);
    colsum_part_kernel<<<dim3((unsigned)blocks, (C + 255) / 256), 256, 0, st>>>(x, part, rows, C);
    DMD_LAUNCH_OK();
    colsum_reduce_kernel<<<(Creal + 255) / 256, 256, 0, st>>>(part, (int)blocks, C, Creal, out, out2, inv);
    DMD_LAUNCH_OK();
    return 0;
  }
  colsum_kernel<<<dim3((unsigned)blocks, (C + 255) / 256), 256, 0, st>>>(x, out, out2, inv, rows, C, Creal);
  DMD_LAUNCH_OK();
  return 0;
}

// norm + SiLU backward, pass 1 (per-channel sums) or pass 2 (gx).  Pixels per block: halved from the whole image until the
// grid covers the SMs twice, but never below 32 pixels
static int norm_bwd_ppb(int B, int HW) {
  int ppb = HW;
  while (ppb > 32 && (long long)B * ((HW + ppb - 1) / ppb) < 2 * kPlanSms) ppb >>= 1;
  return ppb;
}
// det (deterministic mode): pass 1 runs one block per image, so each per-(image, channel) sum has one writer, whose single
// atomic add onto the cleared sum is exact and order-free
static int norm_bwd_launch(const NormBwdParams& nb, int pass, cudaStream_t st, bool det = false) {
  const int ppb = det && pass == 1 ? nb.HW : norm_bwd_ppb(nb.B, nb.HW);
  const dim3 grid((nb.HW + ppb - 1) / ppb, nb.B);
  if (pass == 1) norm_bwd_pass1_kernel<<<grid, kNormThreads, 0, st>>>(nb, ppb);
  else norm_bwd_pass2_kernel<<<grid, kNormThreads, 0, st>>>(nb, ppb);
  DMD_LAUNCH_OK();
  return 0;
}
static int affine_param_grad_launch(const NormBwdParams& nb, float* dgamma, float* dbeta, const float* inv, cudaStream_t st) {
  affine_param_grad_kernel<<<(nb.C + 127) / 128, 128, 0, st>>>(nb.sumA, nb.sumB, nb.B, nb.C, nb.sum_stride, dgamma, dbeta, inv);
  DMD_LAUNCH_OK();
  return 0;
}

// strided SGEMM; chunks > 1 splits K into 16-aligned ranges whose partial products (splitk_partial_floats of `partial`) are
// reduced in a fixed order.  The split count is ceil(K / kchunk), which can be fewer than `chunks`.
static void splitk_plan(int K, int chunks, int* kchunk, int* splits) {
  *kchunk = ((K + chunks - 1) / chunks + 15) / 16 * 16;
  *splits = (K + *kchunk - 1) / *kchunk;
}
// split count of dcond = dfilm Wf over `rows` FiLM rows: K chunks of at least 256 rows, at most 32 (28 for the default net)
static int film_splits(int rows) { return rows / 256 < 32 ? rows / 256 : 32; }
// dcond's split count may be capped by the partials the backward temporary tA holds, down to this many; below it the partials
// get their own buffer.  Every net that trains at cond_channels <= 256 holds at least 8 (its bottom level is an 8 x 8 attention
// level of >= 32 channels: tA >= B x 64 x 32 >= 8 x B x cond_channels floats), so those plans are capped as before.
constexpr int kMinFilmSplits = 8;
static long long splitk_partial_floats(int M, int N, int K, int chunks) {
  if (chunks <= 1) return 0;
  int kchunk, splits;
  splitk_plan(K, chunks, &kchunk, &splits);
  return (long long)splits * M * N;
}
static int sgemm_launch(const float* A, long long sam, long long sak, const float* Bm, long long sbk, long long sbn, float* C, long long ldc,
                        int M, int N, int K, const float* alpha, int accumulate, int chunks, float* partial, cudaStream_t st) {
  if (chunks > 1) {
    DMD_CHECK(ldc == N && partial, "sgemm: split-K needs a dense result (ldc == N) and a partial buffer");
    int kchunk, splits;
    splitk_plan(K, chunks, &kchunk, &splits);
    const long long count = (long long)M * N;
    sgemm_kernel<<<dim3((N + 63) / 64, (M + 63) / 64, splits), 256, 0, st>>>(A, sam, sak, Bm, sbk, sbn, partial, N, M, N, K, nullptr, 0, kchunk, count);
    DMD_LAUNCH_OK();
    splitk_reduce_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(partial, splits, count, C, alpha, accumulate);
    DMD_LAUNCH_OK();
    return 0;
  }
  sgemm_kernel<<<dim3((N + 63) / 64, (M + 63) / 64), 256, 0, st>>>(A, sam, sak, Bm, sbk, sbn, C, ldc, M, N, K, alpha, accumulate);
  DMD_LAUNCH_OK();
  return 0;
}

// attention backward: one CTA per image, the recomputed forward and its gradients in dynamic shared memory
static size_t attn_bwd_smem(int L, int C) {
  return sizeof(float) * ((size_t)L * (C + 1) * 4 + (size_t)L * (3 * C + 4) * 2 + (size_t)(C / 8) * L * 3);
}
// L = 64 runs the instantiation with a compile-time token count, 1 <= L < 64 the one that reads it from ab.L
static int attn_bwd_launch(const AttnBwdParams& ab, int B, cudaStream_t st) {
  DMD_CHECK((ab.C == 64 || ab.C == 32) && ab.L >= 1 && ab.L <= kAttnL && ab.gs > 0 && ab.C % ab.gs == 0 && ab.C / ab.gs <= 4,
            "attention backward: unsupported shape L=%d C=%d gs=%d (1 <= L <= %d)", ab.L, ab.C, ab.gs, kAttnL);
  const size_t smem = attn_bwd_smem(ab.L, ab.C);
  if (ab.L == kAttnL) {
    if (ab.C == 64) attn_bwd_kernel<64, kAttnL><<<B, kAttnThreads, smem, st>>>(ab);
    else attn_bwd_kernel<32, kAttnL><<<B, kAttnThreads, smem, st>>>(ab);
  } else {
    if (ab.C == 64) attn_bwd_kernel<64, 0><<<B, kAttnThreads, smem, st>>>(ab);
    else attn_bwd_kernel<32, 0><<<B, kAttnThreads, smem, st>>>(ab);
  }
  DMD_LAUNCH_OK();
  return 0;
}

static int film_wgrad_launch(const float* dfilm, const float* cond, float* grads, const long long* woff, const long long* boff,
                             int B, int rows, int CC, const float* inv, cudaStream_t st) {
  if (CC <= 256) film_wgrad_kernel<false><<<(rows + 7) / 8, 256, 0, st>>>(dfilm, cond, grads, woff, boff, B, rows, CC, inv);
  else film_wgrad_kernel<true><<<dim3((rows + 7) / 8, (CC + 255) / 256), 256, 0, st>>>(dfilm, cond, grads, woff, boff, B, rows, CC, inv);
  DMD_LAUNCH_OK();
  return 0;
}
static int embedding_bwd_launch(const float* de, const int64_t* act, float* dE, int B, int CC, int T, int num_actions, const float* inv,
                                cudaStream_t st, bool det = false) {
  if (det) embedding_bwd_det_kernel<<<(num_actions * (CC / T) + 255) / 256, 256, 0, st>>>(de, act, dE, B, CC, T, num_actions, inv);
  else embedding_bwd_kernel<<<(B * CC + 255) / 256, 256, 0, st>>>(de, act, dE, B, CC, T, num_actions, inv);
  DMD_LAUNCH_OK();
  return 0;
}
// H, W: the pooled (output) size
static int sumpool2_launch(const float* in, float* out, int B, int H, int W, int C, int accumulate, cudaStream_t st) {
  const long long total4 = (long long)B * H * W * C / 4;
  sumpool2_kernel<<<(unsigned)((total4 + 255) / 256), 256, 0, st>>>(in, out, H, W, C, accumulate, total4);
  DMD_LAUNCH_OK();
  return 0;
}
static int dsilu_mul_launch(const float* pre, const float* dh, float* out, long long n, cudaStream_t st) {
  dsilu_mul_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(pre, dh, out, n);
  DMD_LAUNCH_OK();
  return 0;
}
// H, W: the pre-pool size
static int maxpool2_bwd_launch(const float* y, const float* gp, float* gy, int B, int H, int W, int C, cudaStream_t st) {
  DMD_CHECK(H >= 2 && W >= 2, "maxpool2_bwd: H=%d, W=%d must be at least 2", H, W);
  const int total = (H / 2) * (W / 2) * C;
  maxpool2_bwd_kernel<<<dim3((total + 255) / 256, B), 256, 0, st>>>(y, gp, gy, H, W, C);
  DMD_LAUNCH_OK();
  return 0;
}
static int lstm_cell_bwd_launch(const float* gates, const float* c_in, const float* g_h, const float* g_c, float* dgates, float* g_c_in,
                                int B, int Hd, cudaStream_t st) {
  lstm_cell_bwd_kernel<<<(B * Hd + 255) / 256, 256, 0, st>>>(gates, c_in, g_h, g_c, dgates, g_c_in, B, Hd);
  DMD_LAUNCH_OK();
  return 0;
}
// actor / critic heads: g_h, and the actor bias (dba) / critic weight and bias (dWc, dbc) gradients of the non-null head gradients
static int heads_bwd_launch(const float* g_hx, const float* g_logits, const float* g_val, const float* hx_out, const float* Wa, const float* Wc,
                            float* g_h, float* dba, float* dWc, float* dbc, int B, int Hd, int A, cudaStream_t st) {
  heads_bwd_kernel<<<(B * Hd + 255) / 256, 256, 0, st>>>(g_hx, g_logits, g_val, Wa, Wc, g_h, B, Hd, A);
  DMD_LAUNCH_OK();
  if (g_logits) {
    small_colsum_kernel<<<(A + 31) / 32, 32, 0, st>>>(g_logits, B, A, dba);   // A need not be a multiple of 4
    DMD_LAUNCH_OK();
  }
  if (g_val) {
    vec_outer_sum_kernel<<<(Hd + 127) / 128, 128, 0, st>>>(g_val, hx_out, dWc, dbc, B, Hd);
    DMD_LAUNCH_OK();
  }
  return 0;
}

// ---- per-op entry points of the backward kernels (include/diamond_b200.h): validate, then the launchers above
static int norm_bwd_params(const dmd_norm_bwd_desc* d, NormBwdParams* nb) {
  DMD_CHECK(d && d->x && d->gy && d->stats && d->sumA && d->sumB, "norm_bwd: null argument");
  DMD_CHECK(d->B > 0 && d->HW > 0 && d->C > 0 && d->C % 4 == 0 && d->C <= kMaxCin, "norm_bwd: C=%d must be a positive multiple of 4, <= %d", d->C, kMaxCin);
  DMD_CHECK(d->gs > 0 && d->gs % 4 == 0 && d->C % d->gs == 0 && d->C / d->gs <= 8, "norm_bwd: bad group size %d for C=%d", d->gs, d->C);
  DMD_CHECK(d->mode == 1 ? (d->film != nullptr && d->c_off + d->C <= d->film_ctot) : (d->mode == 2 && d->gamma && d->beta),
            "norm_bwd: mode %d needs %s", d->mode, d->mode == 1 ? "film with c_off + C <= film_ctot" : "gamma and beta (mode 1 or 2)");
  DMD_CHECK(d->sum_stride >= d->C, "norm_bwd: sum_stride %d < C %d", d->sum_stride, d->C);
  NormBwdParams p;
  p.x = d->x; p.gy = d->gy; p.stats = d->stats; p.B = d->B; p.HW = d->HW; p.C = d->C; p.gs = d->gs; p.mode = d->mode; p.act = d->act;
  p.film = d->film; p.film_stride = d->film_stride; p.film_off = d->film_off; p.film_ctot = d->film_ctot; p.c_off = d->c_off;
  p.gamma = d->gamma; p.beta = d->beta; p.eps = d->eps; p.sumA = d->sumA; p.sumB = d->sumB; p.sum_stride = d->sum_stride;
  p.gx = d->gx; p.addend = d->addend; p.accumulate = d->accumulate;
  *nb = p;
  return 0;
}
extern "C" int dmd_norm_bwd(const dmd_norm_bwd_desc* d, int pass, void* stream) {
  NormBwdParams nb;
  if (norm_bwd_params(d, &nb)) return 1;
  DMD_CHECK(pass == 1 || (pass == 2 && d->gx), "norm_bwd: pass must be 1 or 2 (pass 2 writes gx)");
  return norm_bwd_launch(nb, pass, (cudaStream_t)stream);
}
extern "C" int dmd_norm_bwd_det(const dmd_norm_bwd_desc* d, int pass, void* stream) {
  NormBwdParams nb;
  if (norm_bwd_params(d, &nb)) return 1;
  DMD_CHECK(pass == 1 || (pass == 2 && d->gx), "norm_bwd_det: pass must be 1 or 2 (pass 2 writes gx)");
  return norm_bwd_launch(nb, pass, (cudaStream_t)stream, true);
}
extern "C" int dmd_norm_affine_grad(const dmd_norm_bwd_desc* d, float* dgamma, float* dbeta, const float* inv_scale, void* stream) {
  NormBwdParams nb;
  if (norm_bwd_params(d, &nb)) return 1;
  DMD_CHECK(dgamma && dbeta, "norm_affine_grad: null dgamma / dbeta");
  return affine_param_grad_launch(nb, dgamma, dbeta, inv_scale, (cudaStream_t)stream);
}
extern "C" int dmd_attn_bwd(const float* x, const double* stats_in, const float* gamma, const float* beta, const float* wqkv,
                            const float* bqkv, const float* wout, const float* gout, float* gx, float* dgamma, float* dbeta, float* dwqkv,
                            float* dbqkv, float* dwout, float* dbout, const float* inv_scale, int B, int L, int C, int gs, float eps,
                            void* stream) {
  DMD_CHECK(x && stats_in && gamma && beta && wqkv && bqkv && wout && gout && gx && dgamma && dbeta && dwqkv && dbqkv && dwout && dbout,
            "attn_bwd: null argument");
  if (init_kernels()) return 1;
  AttnBwdParams ab{x, stats_in, gamma, beta, wqkv, bqkv, wout, gout, gx, dgamma, dbeta, dwqkv, dbqkv, dwout, dbout, inv_scale, L, C, gs, eps};
  return attn_bwd_launch(ab, B, (cudaStream_t)stream);
}
extern "C" long long dmd_sgemm_partial_floats(int M, int N, int K, int chunks) { return splitk_partial_floats(M, N, K, chunks); }
extern "C" int dmd_sgemm(const float* A, long long sam, long long sak, const float* Bm, long long sbk, long long sbn, float* C, long long ldc,
                         int M, int N, int K, const float* alpha, int accumulate, int chunks, float* partial, void* stream) {
  DMD_CHECK(A && Bm && C && M > 0 && N > 0 && K > 0 && ldc >= N, "sgemm: bad arguments");
  return sgemm_launch(A, sam, sak, Bm, sbk, sbn, C, ldc, M, N, K, alpha, accumulate, chunks, partial, (cudaStream_t)stream);
}
extern "C" int dmd_film_wgrad(const float* dfilm, const float* cond, float* grads, const long long* woff, const long long* boff, int B, int rows,
                              int CC, const float* inv_scale, void* stream) {
  DMD_CHECK(dfilm && cond && grads && woff && boff && B > 0 && rows > 0 && CC > 0 && CC <= kMaxCondChannels,
            "film_wgrad: bad arguments (CC <= %d)", kMaxCondChannels);
  return film_wgrad_launch(dfilm, cond, grads, woff, boff, B, rows, CC, inv_scale, (cudaStream_t)stream);
}
extern "C" int dmd_embedding_bwd(const float* de, const int64_t* act, float* dE, int B, int CC, int T, int num_actions, const float* inv_scale,
                                 void* stream) {
  DMD_CHECK(de && act && dE && B > 0 && T > 0 && CC % T == 0 && num_actions > 0, "embedding_bwd: bad arguments");
  return embedding_bwd_launch(de, act, dE, B, CC, T, num_actions, inv_scale, (cudaStream_t)stream);
}
extern "C" int dmd_embedding_bwd_det(const float* de, const int64_t* act, float* dE, int B, int CC, int T, int num_actions,
                                     const float* inv_scale, void* stream) {
  DMD_CHECK(de && act && dE && B > 0 && T > 0 && CC % T == 0 && num_actions > 0, "embedding_bwd_det: bad arguments");
  return embedding_bwd_launch(de, act, dE, B, CC, T, num_actions, inv_scale, (cudaStream_t)stream, true);
}
extern "C" int dmd_colsum(const float* x, float* out, float* out2, const float* inv_scale, long long rows, int C, int Creal, void* stream) {
  DMD_CHECK(x && out && rows > 0 && C > 0 && C % 4 == 0 && Creal <= C, "colsum: bad arguments (C a multiple of 4, Creal <= C)");
  return colsum_launch(x, out, out2, inv_scale, rows, C, Creal, (cudaStream_t)stream);
}
extern "C" size_t dmd_colsum_partial_bytes(long long rows, int C) { return rows > 0 && C > 0 ? colsum_partial_bytes(rows, C) : 0; }
extern "C" int dmd_colsum_det(const float* x, float* out, float* out2, const float* inv_scale, long long rows, int C, int Creal,
                              void* partial, size_t partial_bytes, void* stream) {
  DMD_CHECK(x && out && partial && rows > 0 && C > 0 && C % 4 == 0 && Creal <= C, "colsum_det: bad arguments (C a multiple of 4, Creal <= C)");
  return colsum_launch(x, out, out2, inv_scale, rows, C, Creal, (cudaStream_t)stream, (float*)partial, partial_bytes);
}
extern "C" int dmd_sumpool2(const float* in, float* out, int B, int H, int W, int C, int accumulate, void* stream) {
  DMD_CHECK(in && out && B > 0 && H > 0 && W > 0 && C % 4 == 0, "sumpool2: bad arguments (C a multiple of 4)");
  return sumpool2_launch(in, out, B, H, W, C, accumulate, (cudaStream_t)stream);
}
extern "C" int dmd_dsilu_mul(const float* pre, const float* dh, float* out, long long n, void* stream) {
  DMD_CHECK(pre && dh && out && n > 0, "dsilu_mul: bad arguments");
  return dsilu_mul_launch(pre, dh, out, n, (cudaStream_t)stream);
}
extern "C" int dmd_maxpool2_bwd(const float* y, const float* gp, float* gy, int B, int H, int W, int C, void* stream) {
  DMD_CHECK(y && gp && gy && B > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C > 0, "maxpool2_bwd: bad arguments (even H, W)");
  return maxpool2_bwd_launch(y, gp, gy, B, H, W, C, (cudaStream_t)stream);
}
extern "C" int dmd_lstm_cell_bwd(const float* gates, const float* c_in, const float* g_h, const float* g_c, float* dgates, float* g_c_in,
                                 int B, int Hd, void* stream) {
  DMD_CHECK(gates && c_in && dgates && g_c_in && B > 0 && Hd > 0, "lstm_cell_bwd: bad arguments");
  return lstm_cell_bwd_launch(gates, c_in, g_h, g_c, dgates, g_c_in, B, Hd, (cudaStream_t)stream);
}
extern "C" int dmd_heads_bwd(const float* g_hx, const float* g_logits, const float* g_val, const float* hx_out, const float* Wa,
                             const float* Wc, float* g_h, float* dba, float* dWc, float* dbc, int B, int Hd, int A, void* stream) {
  DMD_CHECK(Wa && Wc && g_h && B > 0 && Hd > 0 && A > 0, "heads_bwd: bad arguments");
  DMD_CHECK(!g_logits || dba, "heads_bwd: g_logits needs dba");
  DMD_CHECK(!g_val || (hx_out && dWc && dbc), "heads_bwd: g_val needs hx_out, dWc, dbc");
  return heads_bwd_launch(g_hx, g_logits, g_val, hx_out, Wa, Wc, g_h, dba, dWc, dbc, B, Hd, A, (cudaStream_t)stream);
}
extern "C" int dmd_loss_scale(const float* g, long long n, unsigned int* amax, float* scale, void* stream) {
  DMD_CHECK(g && amax && scale && n > 0, "loss_scale: bad arguments");
  return loss_scale_launch(g, n, amax, scale, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------- denoiser executor
// zero-pad / crop copy of an NHWC tensor, then the GroupNorm partial sums of the result (the consumer's prologue reads them)
static int resize_launch(const ResizeParams& p, cudaStream_t st, bool det = false) {
  const long long total = (long long)p.B * p.Hd * p.Wd * (p.C / 4);
  long long blocks = (total + 255) / 256;
  if (blocks > kPlanSms * 16) blocks = kPlanSms * 16;
  resize_nhwc_kernel<<<(int)blocks, 256, 0, st>>>(p);
  DMD_LAUNCH_OK();
  if (p.stats) return gn_stats_launch(p.dst, p.stats, p.B, p.Hd * p.Wd, p.C, p.gs, det, st);
  return 0;
}
extern "C" int dmd_resize_nhwc(const float* src, float* dst, int B, int Hs, int Ws, int Hd, int Wd, int C, double* stats, int gs, void* stream) {
  DMD_CHECK(src && dst && B > 0 && Hs > 0 && Ws > 0 && Hd > 0 && Wd > 0 && C > 0 && C % 4 == 0, "resize_nhwc: bad arguments (C a multiple of 4)");
  DMD_CHECK(!stats || (gs > 0 && C % gs == 0), "resize_nhwc: statistics need C %% gs == 0 (C=%d gs=%d)", C, gs);
  ResizeParams p{src, dst, B, Hs, Ws, Hd, Wd, C, stats, gs};
  return resize_launch(p, (cudaStream_t)stream);
}

namespace {

constexpr float kGnEps = 1e-5f;  // blocks.py:13

// Packed weights the conv kernel keeps resident next to its slab ring: the 128 -> 64 and 64 -> 128 3x3 convs (144 KB) fit
// at the widths the 64-channel nets run, a 128 -> 128 3x3 conv (288 KB) does not
constexpr size_t kResidentWeightMax = 144 * 1024;
constexpr int kMaxConvChunks = 4;   // 256 input channels (a 128-channel level's up-path concat) in chunks of 64
// input channels [c_off, c_off + C) of concat source src, their pack, and (three-pass chunks) their low-part pack
struct ConvChunk { int src, c_off, C; size_t pk_off, pk_lo_off; };
struct ConvW {          // one nn.Conv2d
  int w_idx, b_idx;     // indices into the state_dict pointer list
  int Cout, CoutPad, CinReal, Cin, taps, c0_real, c0_store;
  int precise = 0;      // split-fp16 in one launch: K = 3 * Cin
  int three_pass = 0;   // split-fp16 as three launches (A_hi W_hi, A_lo W_hi, A_hi W_lo): 3 * Cin weights would crowd out the slab ring
  size_t pk_off;        // byte offset into the packed-weight buffer
  size_t pk_lo_off = 0; // three_pass: the low-part pack
  // K split: more than kMaxCin input channels, or weights over kResidentWeightMax, run as one launch per chunk of input
  // channels (each with its own pack at chunk[j].pk_off; pk_off is then unused), accumulating into the output in place.
  // With three_pass, each chunk runs as three passes (its low-part pack at chunk[j].pk_lo_off; pk_lo_off is then unused)
  int nchunks = 0; ConvChunk chunk[kMaxConvChunks] = {};
  // backward-data packs (transposed, tap-flipped; one per source of a channel concat), training only.  A pack over more than
  // kResidentWeightMax bytes is split the same way, over the gradient channels: widthT channels per chunk, one pack each at
  // pkTc_off[k][j] (pkT_off[k] is then unused)
  int nsrcT = 0; int srcC[2] = {0, 0}; int srcOff[2] = {0, 0}; size_t pkT_off[2] = {0, 0};
  int widthT = 0; size_t pkTc_off[2][kMaxConvChunks] = {};
};
struct FilmW { int w_idx, b_idx, C, off; };  // AdaGroupNorm.linear ; off = row offset into the batched FiLM GEMM
struct ResBlockW {
  int cin, cout;
  int has_proj; ConvW proj;
  FilmW n1, n2; ConvW c1, c2;
  int has_attn; int an_w, an_b, qkv_w, qkv_b, op_w, op_b;
};

struct Tens { float* data; double* stats; int C, H, W, gs; float* grad = nullptr; int gid = -1; };

enum OpKind { OP_CONV = 0, OP_ATTN = 1, OP_PREP = 2, OP_RESIZE = 4, OP_STATS = 5 };
struct StatsOp { const float* x; double* stats; int HW, C, gs; };   // GroupNorm partial sums of x (dmd_gn_stats)
struct Op { int kind; ConvParams conv; size_t smem; int cols; AttnParams attn; PrepParams prep; int prep_nsrc; ResizeParams rs; StatsOp gn; };
constexpr int kScratchSlots = 10;  // round-robin pool of PLC16 operand buffers (each lives from its prep to the next conv)

// PLC16 operands produced by one prep launch (op = index of that launch in Plan::ops, replayed by the backward pass)
struct Operand {
  uint8_t *n0 = nullptr, *n1 = nullptr, *r0 = nullptr, *r1 = nullptr, *nl0 = nullptr, *rl0 = nullptr, *rl1 = nullptr; int C0 = 0, C1 = 0, H = 0, W = 0, op = -1;
  // description of the transform (always filled)
  Tens a{}, b{}; bool has_b = false;
  int upsample = 0, mode = 0; const FilmW* film = nullptr; int gamma_idx = 0, beta_idx = 0; bool silu = false, also_raw = false, split = false;
};

// backward op list (training).  Parameter-gradient destinations are OFFSETS into the caller's flat gradient buffer.
enum BKind { B_PREP = 0, B_CONV, B_WGRAD, B_COLSUM, B_NORM1, B_NORM2, B_AFFINE, B_POOL, B_ATTN, B_MEMSET, B_SGEMM, B_FILMW,
             B_LINEAR, B_DSILU, B_EMB, B_ATTN_RECOMP, B_ATTN_CORE };
struct BOp {
  int kind = 0;
  PrepParams prep; int prep_nsrc = 1;
  ConvParams conv; size_t smem = 0; int cols = 0;
  WgradLaunch wg;
  long long goff = -1, goff2 = -1;            // flat-gradient offsets (floats)
  NormBwdParams nb;
  int chunks = 0;                             // sgemm: split-K chunk count (<= 1: no split)
  float* part = nullptr;                      // sgemm: split-K partial buffer (nullptr: tA)
  const float* src = nullptr; float* dst = nullptr; long long rows = 0; int C = 0, Creal = 0, H = 0, W = 0, acc = 0;
  AttnBwdParams ab; long long goffs[6] = {-1, -1, -1, -1, -1, -1};
  // split attention backward (C = 128): ap recomputes q | k | v into ap.scratch; the buffers of attn_core_bwd_kernel
  AttnParams ap; float *at_xn = nullptr, *at_gy = nullptr, *at_y = nullptr, *at_gqkv = nullptr, *at_gxn = nullptr;
  void* ms_ptr = nullptr; size_t ms_bytes = 0;
  // sgemm: C = alpha * op(A) op(B); c_goff >= 0 -> C lives in the gradient buffer
  const float *ga = nullptr, *gb = nullptr; float* gc = nullptr; long long sam = 0, sak = 0, sbk = 0, sbn = 0, ldc = 0, c_goff = -1;
  int M = 0, N = 0, K = 0, use_inv = 0;
  // linear recompute
  const float *lin_in = nullptr, *lin_w = nullptr, *lin_b = nullptr; float* lin_out = nullptr; int lin_K = 0, lin_F = 0;
  // embedding: actions per row (the row's CC channels are T embeddings side by side) and the table's row count
  int emb_T = 0, emb_actions = 0;
};

enum RecKind { R_CONVIN = 0, R_DOWN, R_UP, R_RES, R_OUT };
struct Rec {
  int kind = 0;
  const ConvW* cw = nullptr; const ResBlockW* rb = nullptr;
  Tens x, skip, t, o, a; bool has_skip = false;
  Operand in1, in2;
};

struct Plan {
  int B = 0, H = 0, W = 0;
  int T = 1;   // time-major plans (reward / termination): B = T x segments rows
  bool det = false;   // deterministic mode (torch.use_deterministic_algorithms): fixed-order statistics and gradient sums
  long long tmp_floats = 0;   // training: floats in each of tA / tB / tC
  uint8_t* base = nullptr;
  size_t bytes = 0;
  float *xin = nullptr, *cs = nullptr, *cemb = nullptr, *chid = nullptr, *cond = nullptr, *film = nullptr, *fout = nullptr;
  double* stats = nullptr; size_t stats_bytes = 0;
  int CP_in = 0, CF = 0;
  std::vector<Op> ops;
  uint8_t* scratch[kScratchSlots] = {nullptr};
  int scratch_next = 0;
  // training (dmd_inner_model_forward_train / dmd_denoiser_backward): gradient buffers and the backward op list
  bool train = false;
  int n_grad_tensors = 0;
  std::vector<BOp> bops;
  std::vector<Rec> tape;
  const int64_t* t_act = nullptr;                         // the forward's action tensor (embedding gradient)
  float *tA = nullptr, *tB = nullptr, *tC = nullptr;      // fp32 NHWC temporaries (largest activation)
  uint8_t *gyA = nullptr, *gyB = nullptr;                 // PLC16 gradient operands
  float *gF = nullptr;                                    // scaled dL/d(model output), NHWC with gF_ch channels
  int gF_ch = 0;                                          // round_up(img_channels, 8): the padded channels are zero
  float *dfilm = nullptr, *nsum = nullptr, *partial = nullptr, *scale = nullptr;
  size_t partial_bytes = 0;   // wgrad split-K partials; between weight gradients, the deterministic colsum partials
  float *dcond = nullptr, *dh = nullptr, *cpre = nullptr, *dpre = nullptr, *de = nullptr;
  float* film_part = nullptr;                             // split-K partials of dcond = dfilm Wf: tA, or its own buffer
  int film_splits = 0;                                    // dcond's split count (<= 1: no split)
  long long film_part_own = 0;                            // floats of film_part's own buffer (0: the partials live in tA)
  unsigned int* amax = nullptr;
  const long long *film_woff = nullptr, *film_boff = nullptr;   // the model's FiLM gradient offsets (in its packed buffer)
  uint8_t* zero_begin = nullptr; size_t zero_bytes = 0;   // region cleared at the start of every backward (dfilm, sums, amax)
  // reward / termination training: the encoder output and the LSTM / head tape, time-major rows (row = k * segments + n)
  Tens feat{};
  float *gates = nullptr;                                 // [T][b][4D] pre-activation gates of every step
  float *cseq = nullptr, *hseq = nullptr;                 // [T+1][b][D] cell / hidden states; hseq[0] = h_in, hseq + b*D = y
  float *hid = nullptr, *logits_tm = nullptr;             // [T*b][D] silu(head.0(y)), [T*b][5]
  int64_t* act_tm = nullptr;                              // [T*b] actions
  float *g_tm = nullptr, *g_hid = nullptr, *hpre = nullptr, *g_pre = nullptr, *g_y = nullptr, *dgates = nullptr, *gcs = nullptr;
  // sampler state (NCHW fp32): temporaries only -- the frame stack, the actions and the trajectory are used IN PLACE
  float *s_xc = nullptr, *s_x2 = nullptr, *s_d = nullptr;
  float *sig_all = nullptr, *cemb_all = nullptr, *chid_all = nullptr, *cond_all = nullptr, *film_all = nullptr;  // hoisted conditioning
};

constexpr int kMaxSamplerEvals = 24;   // U-Net evaluations per sample() whose conditioning is hoisted (12 Heun / 24 Euler steps)
struct SamplerGraph {
  bool valid = false;
  int B = 0, H = 0, W = 0; void* ws = nullptr; int order = 0; bool has_eps = false;
  const void *obs = nullptr, *act = nullptr, *traj = nullptr, *eps = nullptr, *out = nullptr; StackView sv{};   // graphs bake pointers in
  unsigned long long stamp = 0;
  std::vector<float> sigmas; float churn[4] = {0, 0, 0, 0};
  long long kernels = 0;  // kernel nodes per replay
  cudaGraphExec_t exec = nullptr;
};

// What every model executor owns apart from its layers: the state_dict tensors (element counts, the caller's pointers and
// offsets into the flat gradient buffer) and the packed-weight buffer (conv packs, then the FiLM table of all AdaGroupNorms).
struct ModelCore {
  int n_tensors = 0;
  std::vector<long long> numel, goff;   // per state_dict tensor: element count and offset into the flat gradient buffer
  long long grad_total = 0;
  std::vector<const float*> ptrs;
  uint8_t* packed = nullptr;
  size_t packed_bytes = 0;
  int cond_channels = 0, film_rows = 0;  // FiLM table: film_rows x cond_channels weights, then film_rows biases
  size_t film_w_off = 0, film_b_off = 0;
  // flat-gradient offset of every FiLM row (weights) / element (biases), the index tables of film_wgrad_kernel.  Model
  // constants, so they live in the packed buffer behind the FiLM table (written by set_weights) and not in a training
  // workspace, whose contents the caller may change between steps
  std::vector<FilmW> films;
  std::vector<long long> film_woff_h, film_boff_h;
  size_t film_woff_off = 0, film_boff_off = 0;
  // training plans, one per live training workspace (an autoregressive Denoiser.forward holds several forwards before
  // their backwards run); kept apart from the inference plan so that imagination and training can alternate
  std::vector<std::unique_ptr<Plan>> tplans;
  // deterministic mode (dmd_*_set_deterministic, torch.use_deterministic_algorithms): part of every plan's cache key
  bool det = false;

  const float* P(int idx) const { return ptrs.empty() ? nullptr : ptrs[idx]; }
  // once every tensor is registered: 16-byte aligned gradient slices, and the FiLM table behind the pk bytes of conv packs
  void finish(size_t pk) {
    n_tensors = (int)numel.size();
    goff.assign(n_tensors, 0);
    grad_total = 0;
    for (int i = 0; i < n_tensors; ++i) { goff[i] = grad_total; grad_total += (numel[i] + 3) & ~3ll; }
    film_w_off = pk; pk += (size_t)film_rows * cond_channels * 4; pk = (pk + 255) & ~(size_t)255;
    film_b_off = pk; pk += (size_t)film_rows * 4; pk = (pk + 255) & ~(size_t)255;
    film_woff_h.assign(film_rows, 0); film_boff_h.assign(film_rows, 0);
    for (const FilmW& f : films)
      for (int r = 0; r < 2 * f.C; ++r) { film_woff_h[f.off + r] = goff[f.w_idx] + (long long)r * cond_channels; film_boff_h[f.off + r] = goff[f.b_idx] + r; }
    film_woff_off = pk; pk += (size_t)film_rows * 8; pk = (pk + 255) & ~(size_t)255;
    film_boff_off = pk; pk += (size_t)film_rows * 8; pk = (pk + 255) & ~(size_t)255;
    packed_bytes = pk;
  }
  const uint8_t* film_offsets_at = nullptr;   // the packed buffer the offset tables were last uploaded into
  int upload_film_offsets(cudaStream_t st) {
    if (film_rows == 0) return 0;
    DMD_CUDA(cudaMemcpyAsync(packed + film_woff_off, film_woff_h.data(), (size_t)film_rows * 8, cudaMemcpyHostToDevice, st));
    DMD_CUDA(cudaMemcpyAsync(packed + film_boff_off, film_boff_h.data(), (size_t)film_rows * 8, cudaMemcpyHostToDevice, st));
    film_offsets_at = packed;
    return 0;
  }
  // adopts the caller's tensors (`module`.state_dict() order); *moved: a tensor or the packed buffer is not where it was
  int set_weights(const char* module, const float* const* ptrs_host, int n_ptrs, void* packed_buf, bool* moved) {
    DMD_CHECK(ptrs_host && packed_buf, "set_weights: null argument");
    DMD_CHECK(n_ptrs == n_tensors, "set_weights: expected %d tensors (%s.state_dict order), got %d", n_tensors, module, n_ptrs);
    *moved = packed != (uint8_t*)packed_buf || ptrs.empty() || memcmp(ptrs.data(), ptrs_host, sizeof(float*) * n_ptrs) != 0;
    ptrs.assign(ptrs_host, ptrs_host + n_ptrs);
    packed = (uint8_t*)packed_buf;
    return 0;
  }
  bool ready() const { return !ptrs.empty() && packed; }
};

long long grad_layout(const ModelCore* m, long long* offsets, long long* numels, int n) {
  if (!m || n != m->n_tensors) { fail("grad_layout: expected %d entries", m ? m->n_tensors : 0); return -1; }
  for (int i = 0; i < n; ++i) { if (offsets) offsets[i] = m->goff[i]; if (numels) numels[i] = m->numel[i]; }
  return m->grad_total;
}

// one reward / termination workspace: the encoder plan (plan.B rows on the workspace at plan.base), then the LSTM / head buffers
struct RewEndLayout {
  Plan plan;
  Tens feat{};  // encoder output: NHWC, last level, time-major rows
  float *x_gates = nullptr, *y = nullptr, *hid = nullptr, *logits_tm = nullptr, *hc[2] = {nullptr, nullptr};
};

}  // namespace

struct dmd_denoiser {
  dmd_denoiser_config cfg;
  ModelCore core;
  // state_dict indices
  int i_fourier = 0, i_actemb = 0, i_cp0w = 0, i_cp0b = 0, i_cp2w = 0, i_cp2b = 0, i_normout_w = 0, i_normout_b = 0;
  ConvW conv_in, conv_out;
  std::vector<std::vector<ResBlockW>> d_blocks, u_blocks;
  std::vector<ResBlockW> mid;
  std::vector<ConvW> downs, ups;  // index 0 unused (Identity)
  Plan plan;
  std::vector<SamplerGraph> graphs;     // one per distinct (buffers, ring head): a WorldModelEnv replays T of them round-robin
  unsigned long long graph_clock = 0;
  cudaStream_t cap_stream = nullptr;
  int need_B = 0, need_H = 0, need_W = 0; bool need_det = false; size_t need_bytes = 0;
};

// Reward / termination model (executor below dmd_lambda_returns): the encoder is built from the U-Net's ResBlocks
struct dmd_rew_end {
  dmd_rew_end_config cfg;
  ModelCore core;
  ConvW conv_in;
  std::vector<std::vector<ResBlockW>> blocks;   // per level, then the two attention ResBlocks
  std::vector<ConvW> downs;                     // index 0 unused
  int i_actemb = 0, i_wih = 0, i_whh = 0, i_bih = 0, i_bhh = 0, i_h0w = 0, i_h0b = 0, i_h2w = 0;
  int feat_c = 0, feat_hw = 0;
  RewEndLayout lay;
};

namespace {

struct Walker {  // assigns state_dict indices in module registration order and packed-buffer offsets
  ModelCore* m; size_t pk = 0; int err = 0;
  int next(long long n) { m->numel.push_back(n); return (int)m->numel.size() - 1; }
  size_t take(size_t bytes) { const size_t off = pk; pk = (pk + bytes + 255) & ~(size_t)255; return off; }
  // split: split-fp16 forward (error ~2^-22), in one launch with K = 3 * Cin when those weights take at most 120 KB of shared
  // memory, else in three launches that leave the slab ring its room
  ConvW conv(int cout, int cin_real, int taps, int c0_real, int c0_store, int c1, bool split = false, bool dgrad = true) {
    ConvW c; c.w_idx = next((long long)cout * cin_real * taps); c.b_idx = next(cout);
    c.Cout = cout; c.CoutPad = round_up(cout, 16); c.CinReal = cin_real; c.taps = taps;
    c.c0_real = c0_real; c.c0_store = c0_store; c.Cin = round_up(c0_store + c1, 16);
    const size_t w1 = (size_t)taps * c.Cin * c.CoutPad * 2;
    if (c.Cin > kMaxCin || w1 > kResidentWeightMax) {
      // chunks of at most kMaxCin channels whose weights stay resident; split-fp16 chunks run in one launch each (K = 3 x chunk)
      const int f = split ? 3 : 1;
      const size_t limit = split ? 120 * 1024 : kResidentWeightMax;
      int width = kMaxCin;
      while (width > 16 && (size_t)taps * width * c.CoutPad * 2 * f > limit) width /= 2;
      const int srcw[2] = {c0_store, c1};
      auto nchunks_at = [&](int wd) { return (srcw[0] + wd - 1) / wd + (srcw[1] + wd - 1) / wd; };
      if (split && nchunks_at(width) > kMaxConvChunks) {
        // split-fp16 chunks that would each run in one launch are too narrow here (a 3x3 128 -> 128 conv: 8 chunks of 16).
        // Instead every chunk runs as three passes, with kResidentWeightMax bytes of weights (64 channels at CoutPad 128)
        c.three_pass = 1;
        width = kMaxCin;
        while (width > 16 && (size_t)taps * width * c.CoutPad * 2 > kResidentWeightMax) width /= 2;
      }
      c.precise = split && !c.three_pass;
      for (int k = 0; k < 2; ++k)
        for (int s = 0; s < srcw[k]; s += width) {
          if (c.nchunks == kMaxConvChunks) { err = fail("plan: a %d -> %d conv needs more than %d K-split chunks", cin_real, cout, kMaxConvChunks); return c; }
          ConvChunk& ch = c.chunk[c.nchunks++];
          ch.src = k; ch.c_off = s; ch.C = srcw[k] - s < width ? srcw[k] - s : width;
          ch.pk_off = take((size_t)taps * ch.C * c.CoutPad * 2 * (c.precise ? 3 : 1));
          if (c.three_pass) ch.pk_lo_off = take((size_t)taps * ch.C * c.CoutPad * 2);
        }
    } else {
      c.precise = split && 3 * w1 <= 120 * 1024;
      c.three_pass = split && !c.precise;
      c.pk_off = take(w1 * (c.precise ? 3 : 1));
      if (c.three_pass) c.pk_lo_off = take(w1);
    }
    if (dgrad) {
      c.nsrcT = c1 ? 2 : 1;
      c.srcC[0] = c0_real; c.srcC[1] = c1; c.srcOff[0] = 0; c.srcOff[1] = c0_real;
      int cmaxT = 16;
      for (int k = 0; k < c.nsrcT; ++k) cmaxT = round_up(c.srcC[k], 16) > cmaxT ? round_up(c.srcC[k], 16) : cmaxT;
      if ((size_t)taps * c.CoutPad * cmaxT * 2 > kResidentWeightMax) {
        c.widthT = c.CoutPad;
        while (c.widthT > 16 && (size_t)taps * c.widthT * cmaxT * 2 > kResidentWeightMax) c.widthT /= 2;
        if (c.CoutPad / c.widthT > kMaxConvChunks) { err = fail("plan: the dgrad of a %d -> %d conv needs more than %d chunks", cin_real, cout, kMaxConvChunks); return c; }
        for (int k = 0; k < c.nsrcT; ++k)
          for (int j = 0; j * c.widthT < c.CoutPad; ++j) c.pkTc_off[k][j] = take((size_t)taps * c.widthT * round_up(c.srcC[k], 16) * 2);
      } else {
        for (int k = 0; k < c.nsrcT; ++k) c.pkT_off[k] = take((size_t)taps * round_up(cout, 16) * round_up(c.srcC[k], 16) * 2);
      }
    }
    return c;
  }
  FilmW film(int C) {
    FilmW f; f.w_idx = next((long long)2 * C * m->cond_channels); f.b_idx = next(2 * C);
    f.C = C; f.off = m->film_rows; m->film_rows += 2 * C; m->films.push_back(f); return f;
  }
  // c0/c1: channels of the two concatenated inputs (c1 = 0: single input)
  ResBlockW resblock(int c0, int c1, int cout, bool attn) {
    ResBlockW r; r.cin = c0 + c1; r.cout = cout;
    r.has_proj = (r.cin != cout);
    if (r.has_proj) r.proj = conv(cout, r.cin, 1, c0, c0, c1, true);  // raw residual stream -> split-fp16
    r.n1 = film(r.cin);
    r.c1 = conv(cout, r.cin, 9, c0, c0, c1);
    r.n2 = film(cout);
    r.c2 = conv(cout, cout, 9, cout, cout, 0);
    r.has_attn = attn;
    if (attn) {
      r.an_w = next(cout); r.an_b = next(cout); r.qkv_w = next((long long)3 * cout * cout); r.qkv_b = next(3 * cout);
      r.op_w = next((long long)cout * cout); r.op_b = next(cout);
    }
    return r;
  }
};

int build_structure(dmd_denoiser* h) {
  const dmd_denoiser_config& c = h->cfg;
  const int L = c.num_levels;
  h->core.cond_channels = c.cond_channels;
  Walker w{&h->core};
  // InnerModel.__init__ registration order (inner_model.py:24-42): noise_emb, act_emb, cond_proj, conv_in, unet,
  // norm_out, conv_out.  UNet (blocks.py:183-220): d_blocks, u_blocks, mid_blocks, downsamples, upsamples.
  const long long CC = c.cond_channels;
  h->i_fourier = w.next(CC / 2); h->i_actemb = w.next((long long)c.num_actions * (CC / c.num_steps_conditioning));
  h->i_cp0w = w.next(CC * CC); h->i_cp0b = w.next(CC); h->i_cp2w = w.next(CC * CC); h->i_cp2b = w.next(CC);
  const int cin_real = (c.num_steps_conditioning + 1) * c.img_channels;
  const int cin_store = round_up(cin_real, 16);
  h->conv_in = w.conv(c.channels[0], cin_real, 9, cin_real, cin_store, 0, true, false);  // its input needs no gradient
  h->d_blocks.resize(L);
  for (int i = 0; i < L; ++i) {
    const int c1 = c.channels[i > 0 ? i - 1 : 0], c2 = c.channels[i];
    for (int k = 0; k < c.depths[i]; ++k) h->d_blocks[i].push_back(w.resblock(k == 0 ? c1 : c2, 0, c2, c.attn_depths[i] != 0));
  }
  // u_blocks were built per level i then reversed (blocks.py:199-207,209): module order = level L-1 ... 0
  h->u_blocks.resize(L);
  for (int m = 0; m < L; ++m) {
    const int i = L - 1 - m;
    const int c1 = c.channels[i > 0 ? i - 1 : 0], c2 = c.channels[i];
    const int n = c.depths[i];
    // list_in_channels = [2*c2]*n + [c1+c2] ; list_out = [c2]*n + [c1]; the concat is (x, skip) with x first.
    // x has c2 channels for every block (block n's x is the previous block's output, c2); skips carry c2 except the
    // last one (the level's x_down, c1 channels).
    for (int k = 0; k <= n; ++k) h->u_blocks[m].push_back(w.resblock(c2, k < n ? c2 : c1, k < n ? c2 : c1, c.attn_depths[i] != 0));
  }
  for (int k = 0; k < 2; ++k) h->mid.push_back(w.resblock(c.channels[L - 1], 0, c.channels[L - 1], true));
  h->downs.resize(L); h->ups.resize(L);
  for (int i = 1; i < L; ++i) h->downs[i] = w.conv(c.channels[i - 1], c.channels[i - 1], 9, c.channels[i - 1], c.channels[i - 1], 0);
  for (int m = 1; m < L; ++m) { const int ch = c.channels[L - 1 - m]; h->ups[m] = w.conv(ch, ch, 9, ch, ch, 0); }
  h->i_normout_w = w.next(c.channels[0]); h->i_normout_b = w.next(c.channels[0]);
  h->conv_out = w.conv(c.img_channels, c.channels[0], 9, c.channels[0], c.channels[0], 0);  // split-fp16 here costs 3x on an N=16 conv for 3.2e-4
  h->core.finish(w.pk);
  return w.err;
}

// ---- descriptors shared by the plan builders and the actor-critic's immediate-mode launches
// single-source operand of src [B][Hs][Ws][C]: raw (mode 0; ups = 2: zero insertion, the adjoint of a stride-2 conv) or
// silu(GroupNorm(gamma, beta)) with the statistics `stats` (mode 2); dst_lo: optional low fp16 part
dmd_prep_desc prep_desc(const float* src, int C, int B, int Hs, int Ws, int ups, int mode, const double* stats, const float* gamma,
                        const float* beta, void* dst, void* dst_lo = nullptr) {
  dmd_prep_desc d; memset(&d, 0, sizeof(d));
  d.src0 = src; d.C0 = C; d.B = B; d.Hs = Hs; d.Ws = Ws; d.upsample = ups; d.mode = mode; d.silu = mode ? 1 : 0;
  if (mode) { d.stats0 = stats; d.gs0 = gn_group_size(C); d.gamma = gamma; d.beta = beta; }
  d.eps = kGnEps; d.dst0 = dst; d.dst_lo0 = dst_lo;
  return d;
}
// backward-data for source k of conv cw: out (+)= conv(gy, W_k^T flipped) at H x W; wpk: the pack at cw.pkT_off[k]
dmd_conv_desc dgrad_desc(const ConvW& cw, int k, const void* wpk, const void* gy, int B, int H, int W, float* out, bool accumulate) {
  dmd_conv_desc d; memset(&d, 0, sizeof(d));
  d.src0 = gy; d.C0 = round_up(cw.Cout, 16); d.B = B; d.H = H; d.W = W; d.taps = cw.taps; d.stride = 1;
  d.wpk = wpk; d.Cout = cw.srcC[k]; d.CoutPad = round_up(cw.srcC[k], 16);
  d.out = out; d.residual = accumulate ? out : nullptr;
  return d;
}
// ConvW::three_pass: pass 0 = A_hi W_hi (+ bias, residual), pass 1 = A_lo W_hi, pass 2 = A_hi W_lo, the later two accumulating
// into the output in place; the statistics come with the last.  d: the one-launch conv with the low operand parts in src*_lo
dmd_conv_desc conv_pass(dmd_conv_desc d, int pass, const void* wpk_lo) {
  const void *lo0 = d.src0_lo, *lo1 = d.src1_lo;
  d.precise = 0; d.src0_lo = d.src1_lo = nullptr;
  if (pass == 1) { d.src0 = lo0; d.src1 = lo1; }
  if (pass == 2) d.wpk = wpk_lo;
  if (pass > 0) { d.bias = nullptr; d.residual = d.out; }
  if (pass < 2) d.out_stats = nullptr;
  return d;
}
// every launch of conv cw, given its one-launch description d: d itself, its three split-fp16 passes, or one launch (or three
// passes) per K-split chunk.  Bias and residual go with the first launch, statistics with the last; the later launches
// accumulate into the output in place.  plane: bytes of one PLC16 plane (8 channels) of the operand; pk: pack offset -> pointer
template <class Pk, class Emit>
int for_each_conv_launch(const ConvW& cw, const dmd_conv_desc& d, size_t plane, Pk pk, Emit emit) {
  const int passes = cw.three_pass ? 3 : 1;
  if (!cw.nchunks) {
    for (int pass = 0; pass < passes; ++pass)
      if (emit(cw.three_pass ? conv_pass(d, pass, pk(cw.pk_lo_off)) : d)) return 1;
    return 0;
  }
  for (int j = 0; j < cw.nchunks; ++j) {
    const ConvChunk& ch = cw.chunk[j];
    const uint8_t* hi = (const uint8_t*)(ch.src ? d.src1 : d.src0);
    const uint8_t* lo = (const uint8_t*)(ch.src ? d.src1_lo : d.src0_lo);
    dmd_conv_desc dc = d;
    dc.src0 = hi + (size_t)(ch.c_off / 8) * plane; dc.src0_lo = lo ? lo + (size_t)(ch.c_off / 8) * plane : nullptr;
    dc.src1 = dc.src1_lo = nullptr; dc.C0 = ch.C; dc.C1 = 0;
    dc.wpk = pk(ch.pk_off);
    if (j > 0) { dc.bias = nullptr; dc.residual = dc.out; }
    if (j + 1 < cw.nchunks) dc.out_stats = nullptr;
    for (int pass = 0; pass < passes; ++pass)
      if (emit(cw.three_pass ? conv_pass(dc, pass, pk(ch.pk_lo_off)) : dc)) return 1;
  }
  return 0;
}
// backward-data of source k of conv cw: one launch, or with split transposed packs (ConvW::widthT) one per chunk of gradient
// channels, accumulating in place.  gy: the PLC16 gradient operand at B x H x W
template <class Emit>
int for_each_dgrad_launch(const ConvW& cw, int k, const uint8_t* packed, const uint8_t* gy, int B, int H, int W, float* out,
                          bool accumulate, Emit emit) {
  const int nch = cw.widthT ? cw.CoutPad / cw.widthT : 1;
  const size_t plane = (size_t)plc_geometry(B, H, W).Qalloc * 16;   // one PLC16 plane holds 8 channels
  for (int j = 0; j < nch; ++j) {
    const void* wpk = packed + (cw.widthT ? cw.pkTc_off[k][j] : cw.pkT_off[k]);
    dmd_conv_desc d = dgrad_desc(cw, k, wpk, gy, B, H, W, out, accumulate || j > 0);
    if (cw.widthT) { d.src0 = gy + (size_t)(j * cw.widthT / 8) * plane; d.C0 = cw.widthT; }
    if (emit(d)) return 1;
  }
  return 0;
}
// the weight gradient kernel takes at most 64 gradient and 64 activation channels: one launch per 64 x 64 (Cout, Cin) block.
// gy / act: PLC16 operands at B x H x W with round_up(Cout, 16) / Ca channels; act channel i is input channel ci_off + i
template <class Emit>
int for_each_wgrad_launch(const ConvW& cw, const uint8_t* gy, const uint8_t* act, int Ca, int Cin, int ci_off, int B, int H, int W,
                          float* partial, const float* inv_scale, Emit emit) {
  const int Cg = round_up(cw.Cout, 16);
  const size_t plane = (size_t)plc_geometry(B, H, W).Qalloc * 16;
  for (int co = 0; co < Cg; co += 64)
    for (int ca = 0; ca < Ca; ca += 64) {
      const int cg_n = Cg - co < 64 ? Cg - co : 64, ca_n = Ca - ca < 64 ? Ca - ca : 64;
      const int cout_n = cw.Cout - co < 64 ? cw.Cout - co : 64, cin_n = Cin - ca < 64 ? Cin - ca : 64;
      if (cin_n <= 0) continue;
      WgradLaunch L;
      if (wgrad_fill(gy + (size_t)(co / 8) * plane, cg_n, act + (size_t)(ca / 8) * plane, ca_n, B, H, W, cw.taps, partial, cout_n, cin_n,
                     cw.CinReal, ci_off + ca, inv_scale, 1, &L, co)) return 1;
      if (emit(L)) return 1;
    }
  return 0;
}
// silu(GroupNorm(gamma, beta)) backward of x [B][HW][C] (mode 2): per-channel sums in nsum ([2][B][kMaxCin], zeroed before
// pass 1), gx (+)= the input gradient (+ addend)
NormBwdParams gn_bwd_params(const float* x, const float* gy, const double* stats, int B, int HW, int C, int gs, const float* gamma,
                            const float* beta, float* nsum, float* gx, const float* addend, bool accumulate) {
  NormBwdParams nb; memset(&nb, 0, sizeof(nb));
  nb.x = x; nb.gy = gy; nb.stats = stats; nb.B = B; nb.HW = HW; nb.C = C; nb.gs = gs; nb.mode = 2; nb.act = 1; nb.eps = kGnEps;
  nb.gamma = gamma; nb.beta = beta;
  nb.sumA = nsum; nb.sumB = nsum ? nsum + (size_t)B * kMaxCin : nullptr; nb.sum_stride = kMaxCin;
  nb.gx = gx; nb.addend = addend; nb.accumulate = accumulate ? 1 : 0;
  return nb;
}

struct Bump {
  uint8_t* base; size_t off = 0;
  void* take(size_t bytes) { off = (off + 255) & ~(size_t)255; void* p = base ? base + off : nullptr; off += bytes; return p; }
};

// -- plan construction: mirrors InnerModel.forward / UNet.forward / ResBlock.forward
struct PlanBuilder {
  const ModelCore* core; Plan* pl; Bump* bump; Bump* sbump; int err = 0;

  Tens tensor(int C, int H, int W, bool with_stats, bool with_grad = true) {
    Tens t; t.C = C; t.H = H; t.W = W; t.gs = gn_group_size(C);
    t.data = (float*)bump->take((size_t)pl->B * H * W * C * 4);
    t.stats = with_stats ? (double*)sbump->take((size_t)pl->B * (C / t.gs) * 2 * 8) : nullptr;
    if (pl->train && with_grad) { t.grad = (float*)bump->take((size_t)pl->B * H * W * C * 4); t.gid = pl->n_grad_tensors++; }
    return t;
  }
  void record(const Rec& r) { if (pl->train) pl->tape.push_back(r); }
  const float* P(int idx) const { return core->P(idx); }
  const void* pk(size_t off) const { return core->packed ? core->packed + off : (const void*)1; }

  uint8_t* scratch() {
    uint8_t* p = pl->scratch[pl->scratch_next];
    pl->scratch_next = (pl->scratch_next + 1) % kScratchSlots;
    return p ? p : (uint8_t*)1;
  }

  // mode 0 raw / 1 AdaGroupNorm(film) / 2 GroupNorm(gamma,beta); also_raw: additionally emit the raw operand (skip projection)
  // split: also emit the low fp16 part of the operand that a precise conv will read (raw if also_raw, else the main one)
  Operand prep(const Tens& a, const Tens* b, int upsample, int mode, const FilmW* film, int gamma_idx, int beta_idx, bool silu, bool also_raw, bool split = false) {
    Operand o;
    o.a = a; o.has_b = b != nullptr; if (b) o.b = *b;
    o.upsample = upsample; o.mode = mode; o.film = film; o.gamma_idx = gamma_idx; o.beta_idx = beta_idx; o.silu = silu; o.also_raw = also_raw; o.split = split;
    o.C0 = round_up(a.C, 16); o.C1 = b ? round_up(b->C, 16) : 0;
    o.H = upsample ? 2 * a.H : a.H; o.W = upsample ? 2 * a.W : a.W;
    materialize(o);
    return o;
  }
  void materialize(Operand& o) {
    if (o.n0) return;
    const Tens& a = o.a; const Tens* b = o.has_b ? &o.b : nullptr;
    dmd_prep_desc d; memset(&d, 0, sizeof(d));
    d.src0 = a.data ? a.data : (const float*)1; d.C0 = a.C; d.src1 = b ? (b->data ? b->data : (const float*)1) : nullptr; d.C1 = b ? b->C : 0;
    d.B = pl->B; d.Hs = a.H; d.Ws = a.W; d.upsample = o.upsample; d.mode = o.mode; d.silu = o.silu;
    if (o.mode) {
      d.stats0 = a.stats ? a.stats : (const double*)1; d.gs0 = a.gs;
      if (b) { d.stats1 = b->stats ? b->stats : (const double*)1; d.gs1 = b->gs; }
    }
    if (o.mode == 1) { d.film = pl->film ? pl->film : (const float*)1; d.film_stride = core->film_rows; d.film_off = o.film->off; }
    if (o.mode == 2) { d.gamma = P(o.gamma_idx) ? P(o.gamma_idx) : (const float*)1; d.beta = P(o.beta_idx) ? P(o.beta_idx) : (const float*)1; }
    d.eps = kGnEps;
    o.n0 = scratch(); d.dst0 = o.n0;
    if (b) { o.n1 = scratch(); d.dst1 = o.n1; }
    if (o.also_raw) { o.r0 = scratch(); d.dst_raw0 = o.r0; if (b) { o.r1 = scratch(); d.dst_raw1 = o.r1; } }
    if (o.split && o.also_raw) { o.rl0 = scratch(); d.dst_raw_lo0 = o.rl0; if (b) { o.rl1 = scratch(); d.dst_raw_lo1 = o.rl1; } }
    if (o.split && !o.also_raw) { o.nl0 = scratch(); d.dst_lo0 = o.nl0; }
    Op op; op.kind = OP_PREP;
    if (prep_fill(&d, &op.prep, &op.prep_nsrc)) { err = 1; return; }
    o.op = (int)pl->ops.size();
    pl->ops.push_back(op);
  }

  void conv(const ConvW& cw, Operand& in, bool raw, int stride, const Tens* resid, Tens& out, bool out_stats,
            const ConvW* xproj = nullptr, Operand* xin = nullptr) {
    materialize(in);
    if (xin) materialize(*xin);
    if (err) return;
    dmd_conv_desc d; memset(&d, 0, sizeof(d));
    if (xproj) {  // skip projection of the block input, accumulated into this conv's output tile
      d.xsrc0 = xin->r0; d.xsrc0_lo = xin->rl0; d.xC0 = xin->C0;
      if (xin->C1) { d.xsrc1 = xin->r1; d.xsrc1_lo = xin->rl1; d.xC1 = xin->C1; }
      d.wpk_x = pk(xproj->pk_off); d.bias_x = P(xproj->b_idx);
      if (!xproj->precise) { fail("plan: a fused projection needs its split-fp16 weights in one pack"); err = 1; return; }
    }
    const bool split = cw.precise || cw.three_pass;
    d.src0 = raw ? in.r0 : in.n0; d.src1 = in.C1 ? (raw ? in.r1 : in.n1) : nullptr;
    d.precise = cw.precise;
    if (split) { d.src0_lo = raw ? in.rl0 : in.nl0; d.src1_lo = in.C1 ? in.rl1 : nullptr; }
    d.C0 = in.C0; d.C1 = in.C1; d.B = pl->B; d.H = in.H; d.W = in.W; d.taps = cw.taps; d.stride = stride;
    d.wpk = pk(cw.pk_off); d.bias = P(cw.b_idx);
    d.Cout = cw.Cout; d.CoutPad = cw.CoutPad;
    d.residual = resid ? (resid->data ? resid->data : (const float*)1) : nullptr; d.out = out.data ? out.data : (float*)1;
    d.out_stats = out_stats ? (out.stats ? out.stats : (double*)1) : nullptr; d.out_gs = out.gs;
    // below 7x7, and in deterministic mode, the statistics come from gn_stats over the finished output (the same sums; one
    // launch more)
    const bool stats_after = d.out_stats && (pl->det || !conv_epilogue_stats_fit(in.H, in.W));
    if (stats_after) d.out_stats = nullptr;
    if (split && (!d.src0_lo || (in.C1 && !d.src1_lo))) { fail("plan: precise conv without low operand parts"); err = 1; return; }
    if (in.C0 + in.C1 != cw.Cin) { fail("plan: operand channels %d+%d do not match the packed weights (%d)", in.C0, in.C1, cw.Cin); err = 1; return; }
    if (cw.nchunks && xproj) { fail("plan: a K-split conv cannot carry a fused projection"); err = 1; return; }
    const size_t plane = (size_t)plc_geometry(pl->B, in.H, in.W).Qalloc * 16;   // one PLC16 plane holds 8 channels
    if (for_each_conv_launch(cw, d, plane, [&](size_t off) { return pk(off); }, [&](const dmd_conv_desc& dc) {
      Op op; op.kind = OP_CONV;
      if (conv_fill(&dc, &op.conv, &op.smem, &op.cols)) return 1;
      pl->ops.push_back(op);
      return 0;
    })) err = 1;
    if (stats_after) stats_of(out);
  }
  void stats_of(const Tens& t) {
    Op op; op.kind = OP_STATS;
    op.gn = StatsOp{t.data ? t.data : (const float*)1, t.stats ? t.stats : (double*)1, t.H * t.W, t.C, t.gs};
    pl->ops.push_back(op);
  }

  // ResBlock.forward (blocks.py:141-147)
  Tens resblock(const ResBlockW& rb, const Tens& x, const Tens* skip) {
    const int H = x.H, W = x.W;
    Operand in1 = prep(x, skip, 0, 1, &rb.n1, 0, 0, true, rb.has_proj != 0, rb.has_proj != 0);
    Tens t = tensor(rb.cout, H, W, true, false);   // its gradient lives in a temporary
    conv(rb.c1, in1, false, 1, nullptr, t, true);
    Operand in2 = prep(t, nullptr, 0, 1, &rb.n2, 0, 0, true, false);
    Tens o = tensor(rb.cout, H, W, true);
    // x + r: r is the block input itself, or proj(input) fused into conv2's accumulator (no r tensor, no extra launch).  When
    // either is K-split, proj(input) runs first into o and conv2 accumulates onto it
    if (rb.has_proj && !rb.c2.nchunks && !rb.proj.nchunks) conv(rb.c2, in2, false, 1, nullptr, o, true, &rb.proj, &in1);
    else if (rb.has_proj) { conv(rb.proj, in1, true, 1, nullptr, o, false); conv(rb.c2, in2, false, 1, &o, o, true); }
    else conv(rb.c2, in2, false, 1, &x, o, true);
    Rec rec; rec.kind = R_RES; rec.rb = &rb; rec.x = x; rec.has_skip = skip != nullptr; if (skip) rec.skip = *skip;
    rec.t = t; rec.o = o; rec.in1 = in1; rec.in2 = in2;
    if (!rb.has_attn) { record(rec); return o; }
    if (pl->train && H * W > kAttnL) {
      fail("training: the attention backward (attn_bwd_kernel) is built for at most %d tokens (8x8); this plan has an attention block "
           "over %dx%d = %d tokens (inference runs at any token count)", kAttnL, H, W, H * W);
      err = 1;
      return o;
    }
    Tens a = tensor(rb.cout, H, W, true);
    Op op; op.kind = OP_ATTN;
    op.attn = AttnParams{o.data, o.stats, P(rb.an_w), P(rb.an_b), P(rb.qkv_w), P(rb.qkv_b), P(rb.op_w), P(rb.op_b), a.data, a.stats, H * W, rb.cout, o.gs, kGnEps};
    if (H * W != kAttnL) op.attn.scratch = (float*)bump->take(attn_scratch_bytes(pl->B, H * W, rb.cout));
    if (pl->det) op.attn.ostats = nullptr;
    pl->ops.push_back(op);
    if (pl->det) stats_of(a);
    rec.a = a;
    record(rec);
    return a;
  }

  // RewEndEncoder.forward (rew_end_model.py:127-132): conv_in, then per level [Downsample] + ResBlocks, then two attention
  // ResBlocks; the same blocks as the U-Net, conditioned on the action embedding.  Output: *feat (NHWC, last level).
  int build_rew_end(const dmd_rew_end* h, Tens* feat) {
    const dmd_rew_end_config& c = h->cfg;
    const int L = c.num_levels, B = pl->B, H = pl->H, W = pl->W;
    if (H % (1 << (L - 1)) || W % (1 << (L - 1))) return fail("rew_end: H=%d W=%d must be multiples of %d", H, W, 1 << (L - 1));
    int cmax = 16;
    for (int i = 0; i < L; ++i) cmax = c.channels[i] > cmax ? c.channels[i] : cmax;
    const size_t slot_bytes = (plc16_bytes(B, H, W, cmax) + 255) & ~(size_t)255;
    for (int i = 0; i < kScratchSlots; ++i) pl->scratch[i] = (uint8_t*)bump->take(slot_bytes);
    pl->scratch_next = 0;
    pl->CP_in = h->conv_in.c0_store;
    pl->xin = (float*)bump->take((size_t)B * H * W * pl->CP_in * 4);
    pl->cond = (float*)bump->take((size_t)B * c.cond_channels * 4);
    pl->film = (float*)bump->take((size_t)B * core->film_rows * 4);
    Tens xin{pl->xin, nullptr, pl->CP_in, H, W, 8};
    Tens x = tensor(c.channels[0], H, W, true);
    {
      Operand in0 = prep(xin, nullptr, 0, 0, nullptr, 0, 0, false, false, true);
      conv(h->conv_in, in0, false, 1, nullptr, x, true);
      Rec rec; rec.kind = R_CONVIN; rec.cw = &h->conv_in; rec.x = xin; rec.o = x; rec.in1 = in0; record(rec);
    }
    for (int i = 0; i <= L; ++i) {
      if (i > 0 && i < L) {
        Tens xd = tensor(c.channels[i - 1], x.H / 2, x.W / 2, true);
        Operand ind = prep(x, nullptr, 0, 0, nullptr, 0, 0, false, false);
        conv(h->downs[i], ind, false, 2, nullptr, xd, true);
        Rec rec; rec.kind = R_DOWN; rec.cw = &h->downs[i]; rec.x = x; rec.o = xd; rec.in1 = ind; record(rec);
        x = xd;
      }
      for (auto& rb : h->blocks[i]) x = resblock(rb, x, nullptr);
    }
    *feat = x;
    return err;
  }

  void resize(const Tens& src, const Tens& dst) {
    Op op; op.kind = OP_RESIZE;
    op.rs = ResizeParams{src.data ? src.data : (const float*)1, dst.data ? dst.data : (float*)1, pl->B, src.H, src.W, dst.H, dst.W, src.C,
                         dst.stats ? dst.stats : (double*)1, dst.gs};
    pl->ops.push_back(op);
  }

  int build(const dmd_denoiser* h) {
    const dmd_denoiser_config& c = h->cfg;
    const int L = c.num_levels, B = pl->B, H = pl->H, W = pl->W;
    const int div = 1 << (L - 1);
    // UNet.forward pads its input (the conv_in output) at the bottom / right to multiples of 2^(levels-1) and crops its output
    // back (blocks.py:225-229,245): conv_in and norm_out / conv_out run at H x W, everything between at Hp x Wp
    const int Hp = (H + div - 1) / div * div, Wp = (W + div - 1) / div * div;
    const bool padded = Hp != H || Wp != W;
    if (padded && pl->train) return fail("denoiser: training at H=%d W=%d (not multiples of %d) needs the pad / crop adjoints, which are not built", H, W, div);
    // operand scratch pool: sized for the largest operand of the network (level 0, widest channel count)
    int cmax = 16;
    for (int i = 0; i < L; ++i) cmax = c.channels[i] > cmax ? c.channels[i] : cmax;
    const size_t slot_bytes = (plc16_bytes(B, Hp, Wp, cmax) + 255) & ~(size_t)255;
    for (int i = 0; i < kScratchSlots; ++i) pl->scratch[i] = (uint8_t*)bump->take(slot_bytes);
    pl->scratch_next = 0;
    pl->CP_in = h->conv_in.c0_store;
    pl->xin = (float*)bump->take((size_t)B * H * W * pl->CP_in * 4);
    pl->cs = (float*)bump->take((size_t)(B + 1) * 4 * 4);  // +1: scalar sigma slot used by the sampler
    pl->cemb = (float*)bump->take((size_t)B * c.cond_channels * 4);
    pl->chid = (float*)bump->take((size_t)B * c.cond_channels * 4);
    pl->cond = (float*)bump->take((size_t)B * c.cond_channels * 4);
    pl->film = (float*)bump->take((size_t)B * core->film_rows * 4);
    Tens xin{pl->xin, nullptr, pl->CP_in, H, W, 8};
    Tens x = tensor(c.channels[0], H, W, !padded);
    {
      Operand in = prep(xin, nullptr, 0, 0, nullptr, 0, 0, false, false, true);
      conv(h->conv_in, in, false, 1, nullptr, x, !padded);
      Rec rec; rec.kind = R_CONVIN; rec.cw = &h->conv_in; rec.x = xin; rec.o = x; rec.in1 = in; record(rec);
    }
    if (padded) {
      Tens xp = tensor(c.channels[0], Hp, Wp, true);
      resize(x, xp);
      x = xp;
    }
    std::vector<std::vector<Tens>> d_outputs;
    for (int i = 0; i < L; ++i) {
      Tens xd = x;
      if (i > 0) {  // Downsample (blocks.py:93-100): raw input, stride 2
        xd = tensor(c.channels[i - 1], x.H / 2, x.W / 2, true);
        Operand in = prep(x, nullptr, 0, 0, nullptr, 0, 0, false, false);
        conv(h->downs[i], in, false, 2, nullptr, xd, true);
        Rec rec; rec.kind = R_DOWN; rec.cw = &h->downs[i]; rec.x = x; rec.o = xd; rec.in1 = in; record(rec);
      }
      std::vector<Tens> outs{xd};
      x = xd;
      for (auto& rb : h->d_blocks[i]) { x = resblock(rb, x, nullptr); outs.push_back(x); }
      d_outputs.push_back(outs);
    }
    for (auto& rb : h->mid) x = resblock(rb, x, nullptr);
    for (int m = 0; m < L; ++m) {
      Tens xu = x;
      if (m > 0) {  // Upsample (blocks.py:103-110): nearest x2 folded into the operand, then conv
        xu = tensor(x.C, x.H * 2, x.W * 2, true);
        Operand in = prep(x, nullptr, 1, 0, nullptr, 0, 0, false, false);
        conv(h->ups[m], in, false, 1, nullptr, xu, true);
        Rec rec; rec.kind = R_UP; rec.cw = &h->ups[m]; rec.x = x; rec.o = xu; rec.in1 = in; record(rec);
      }
      x = xu;
      const std::vector<Tens>& skip = d_outputs[L - 1 - m];  // reversed(d_outputs); block k uses skip[::-1][k]
      const int ns = (int)skip.size();
      for (size_t k = 0; k < h->u_blocks[m].size(); ++k) x = resblock(h->u_blocks[m][k], x, &skip[ns - 1 - (int)k]);
    }
    if (padded) {   // x[..., :h, :w]
      Tens xc = tensor(x.C, H, W, true);
      resize(x, xc);
      x = xc;
    }
    pl->CF = c.img_channels;
    pl->fout = (float*)bump->take((size_t)B * H * W * pl->CF * 4);
    Tens f{pl->fout, nullptr, pl->CF, H, W, pl->CF};
    // conv_out(silu(norm_out(x)))  (inner_model.py:48)
    {
      Operand in = prep(x, nullptr, 0, 2, nullptr, h->i_normout_w, h->i_normout_b, true, false, false);
      conv(h->conv_out, in, false, 1, nullptr, f, false);
      Rec rec; rec.kind = R_OUT; rec.cw = &h->conv_out; rec.x = x; rec.in1 = in; record(rec);
    }
    // sampler temporaries + hoisted conditioning of up to kMaxSamplerEvals evaluations
    const size_t img = (size_t)B * c.img_channels * H * W * 4;
    pl->s_xc = (float*)bump->take(img); pl->s_x2 = (float*)bump->take(img); pl->s_d = (float*)bump->take(img);
    if (!pl->train) {
      const size_t K = kMaxSamplerEvals;
      pl->sig_all = (float*)bump->take(K * 4);
      pl->cemb_all = (float*)bump->take(K * B * c.cond_channels * 4); pl->chid_all = (float*)bump->take(K * B * c.cond_channels * 4);
      pl->cond_all = (float*)bump->take(K * B * c.cond_channels * 4); pl->film_all = (float*)bump->take(K * B * core->film_rows * 4);
    }
    return err;
  }
};

int make_plan(const dmd_denoiser* h, Plan* pl, int B, int H, int W, uint8_t* base, size_t* total) {
  pl->B = B; pl->H = H; pl->W = W; pl->ops.clear();
  // pass 1: stats region size (tiny) — run the builder on null bases
  Bump b0{nullptr}, s0{nullptr};
  { Plan tmp; tmp.B = B; tmp.H = H; tmp.W = W; tmp.det = h->core.det; PlanBuilder pb{&h->core, &tmp, &b0, &s0}; if (pb.build(h)) return 1; }
  const size_t stats_bytes = (s0.off + 255) & ~(size_t)255;
  if (total) *total = stats_bytes + b0.off + 256;
  if (!base) return 0;
  Bump sb{base}, bb{base + stats_bytes};
  pl->base = base; pl->stats = (double*)base; pl->stats_bytes = stats_bytes; pl->det = h->core.det;
  PlanBuilder pb{&h->core, pl, &bb, &sb};
  if (pb.build(h)) return 1;
  pl->bytes = stats_bytes + bb.off;
  return 0;
}

// ---------------------------------------------------------------------------------------------- backward plan (training)
// Walks the forward tape in reverse and emits the backward op list.  Every gradient tensor is fp32 NHWC and carries the
// loss scale; "first writer assigns, later writers accumulate" is decided here at plan time (ginit), so no gradient
// buffer needs a memset.  Forward conv inputs (the PLC16 operands) are not kept: the forward prep launch is replayed.
// Both executors' encoders are made of the same records (R_RES, R_DOWN, R_UP, R_CONVIN), which walk() handles; each model
// emits its own output head before the walk and its own conditioning path after it (film_tail is the part they share).
struct BwdBuilder {
  const ModelCore* core; Plan* pl; int err = 0;
  std::vector<char> ginit;

  const float* P(int idx) const { return core->P(idx); }
  long long G(int idx) const { return core->goff[idx]; }
  bool was_init(const Tens& t) { const bool w = ginit[t.gid] != 0; ginit[t.gid] = 1; return w; }
  void push(const BOp& b) { pl->bops.push_back(b); }
  void begin() { ginit.assign(pl->n_grad_tensors, 0); pl->bops.clear(); }

  void replay(const Operand& o) { BOp b; b.kind = B_PREP; b.prep = pl->ops[o.op].prep; b.prep_nsrc = pl->ops[o.op].prep_nsrc; push(b); }
  // NHWC fp32 gradient [B][Hs][Ws][C] -> PLC16 operand (ups = 2: zero insertion, the adjoint of a stride-2 conv)
  void gprep(const float* g, int C, int Hs, int Ws, int ups, uint8_t* dst) {
    const dmd_prep_desc d = prep_desc(g, C, pl->B, Hs, Ws, ups, 0, nullptr, nullptr, nullptr, dst);
    BOp b; b.kind = B_PREP;
    if (prep_fill(&d, &b.prep, &b.prep_nsrc)) { err = 1; return; }
    push(b);
  }
  void colsum(const float* g, long long rows, int C, int Creal, int idx, int idx2 = -1) {
    BOp b; b.kind = B_COLSUM; b.src = g; b.rows = rows; b.C = C; b.Creal = Creal; b.goff = G(idx); b.goff2 = idx2 >= 0 ? G(idx2) : -1;
    push(b);
  }
  // one launch, or with split transposed packs (ConvW::widthT) one per chunk of gradient channels, accumulating in place
  void dgrad(const ConvW& cw, int k, const uint8_t* gy, int H, int W, float* out, bool accumulate) {
    if (for_each_dgrad_launch(cw, k, core->packed, gy, pl->B, H, W, out, accumulate, [&](const dmd_conv_desc& d) {
      BOp b; b.kind = B_CONV;
      if (conv_fill(&d, &b.conv, &b.smem, &b.cols)) return 1;
      push(b);
      return 0;
    })) err = 1;
  }
  void wgrad(const ConvW& cw, const uint8_t* gy, const uint8_t* act, int Ca, int Cin, int ci_off, int H, int W) {
    if (for_each_wgrad_launch(cw, gy ? gy : (const uint8_t*)1, act ? act : (const uint8_t*)1, Ca, Cin, ci_off, pl->B, H, W,
                              pl->partial ? pl->partial : (float*)1, pl->scale ? pl->scale + 1 : (const float*)1, [&](const WgradLaunch& L) {
      BOp b; b.kind = B_WGRAD; b.goff = G(cw.w_idx); b.wg = L;
      push(b);
      return 0;
    })) err = 1;
  }
  void norm_bwd(const Tens& x, const float* gy, int mode, const FilmW* film, int c_off, int ctot, int gamma_idx, int beta_idx,
                float* gx, const float* addend, bool accumulate, bool silu = true) {
    const int R = core->film_rows;
    NormBwdParams nb = gn_bwd_params(x.data, gy, x.stats, pl->B, x.H * x.W, x.C, x.gs, P(gamma_idx), P(beta_idx), pl->nsum, gx, addend, accumulate);
    nb.act = silu ? 1 : 0;
    if (mode == 1) {   // AdaGroupNorm: FiLM rows in place of gamma / beta, their gradients in place of the per-channel sums
      nb.mode = 1; nb.gamma = nb.beta = nullptr; nb.c_off = c_off;
      nb.film = pl->film; nb.film_stride = R; nb.film_off = film->off; nb.film_ctot = ctot;
      nb.sumB = pl->dfilm ? pl->dfilm + film->off + c_off : nullptr;            // d scale
      nb.sumA = pl->dfilm ? pl->dfilm + film->off + ctot + c_off : nullptr;     // d shift
      nb.sum_stride = R;
    } else {
      BOp m; m.kind = B_MEMSET; m.ms_ptr = pl->nsum; m.ms_bytes = (size_t)2 * pl->B * kMaxCin * 4; push(m);
    }
    BOp b1; b1.kind = B_NORM1; b1.nb = nb;
    push(b1);
    if (mode == 2) {
      BOp a; a.kind = B_AFFINE; a.nb = nb; a.goff = G(gamma_idx); a.goff2 = G(beta_idx); push(a);
    }
    BOp b2 = b1; b2.kind = B_NORM2; push(b2);
  }

  // SelfAttention2d backward at C = 128, and at every C in deterministic mode (attn_bwd_kernel adds its parameter gradients
  // with atomics; here they are fixed-order sgemm / colsum launches), L = H * W <= 64 (bwd_kernels.cuh): x = o, g_out = gout,
  // g_x assigned to o.grad.
  // Buffers in tB (q | k | v, g_qkv) and tC (xn, g_y, y, g_xn); the weight-gradient products split K over tA
  void attn_split(const ResBlockW& rb, const Tens& o, const float* gout) {
    const int C = rb.cout, L = o.H * o.W, rows = pl->B * L;
    const long long n = (long long)rows * C;
    if (6 * n > pl->tmp_floats) { err = fail("backward plan: attention temporaries (%lld floats) exceed tB", 6 * n); return; }
    BOp b; b.kind = B_ATTN_RECOMP;
    b.ap = AttnParams{o.data, o.stats, P(rb.an_w), P(rb.an_b), P(rb.qkv_w), P(rb.qkv_b), P(rb.op_w), P(rb.op_b), nullptr, nullptr, L, C, o.gs, kGnEps};
    b.ap.scratch = pl->tB; b.ap.out = const_cast<float*>(gout);   // attn_core_bwd_kernel reads g_out from ap.out
    b.at_gqkv = pl->tB + 3 * n;
    b.at_xn = pl->tC; b.at_gy = pl->tC + n; b.at_y = pl->tC + 2 * n; b.at_gxn = pl->tC + 3 * n;
    push(b);
    sgemm(gout, C, 1, P(rb.op_w), C, 1, b.at_gy, -1, C, rows, C, C, 0, 0);                       // g_y = g_out Wo
    BOp c = b; c.kind = B_ATTN_CORE; push(c);
    sgemm(gout, 1, C, b.at_y, C, 1, nullptr, G(rb.op_w), C, C, C, rows, 1, 1); split_k();        // dWo += g_out^T y
    colsum(gout, rows, C, C, rb.op_b);
    sgemm(b.at_gqkv, 1, 3 * C, b.at_xn, C, 1, nullptr, G(rb.qkv_w), C, 3 * C, C, rows, 1, 1); split_k();   // dWqkv += g_qkv^T xn
    colsum(b.at_gqkv, rows, 3 * C, 3 * C, rb.qkv_b);
    sgemm(b.at_gqkv, 3 * C, 1, P(rb.qkv_w), C, 1, b.at_gxn, -1, C, rows, C, 3 * C, 0, 1);      // g_xn += g_qkv Wqkv
    norm_bwd(o, b.at_gxn, 2, nullptr, 0, C, rb.an_w, rb.an_b, o.grad, nullptr, false, false);
  }
  void split_k() {   // the last sgemm contracts over every token of the batch: split K across the SMs, partials in tA
    BOp& s = pl->bops.back();
    const long long fit = pl->tmp_floats / ((long long)s.M * s.N);
    int splits = s.K / 256; if (splits > 32) splits = 32; if (splits > fit) splits = (int)fit;
    if (splits > 1) s.chunks = splits;
  }

  // ResBlock.forward (blocks.py:141-147) backward
  void resblock(const Rec& r) {
    const ResBlockW& rb = *r.rb;
    const int H = r.o.H, W = r.o.W, B = pl->B;
    const long long pix = (long long)B * H * W;
    Tens o = r.o;
    if (rb.has_attn && (rb.cout > 64 || pl->det)) {
      attn_split(rb, o, r.a.grad);
      ginit[o.gid] = 1;
    } else if (rb.has_attn) {  // attention consumes o alone: its backward ASSIGNS o's gradient
      BOp b; b.kind = B_ATTN;
      b.ab = AttnBwdParams{o.data, o.stats, P(rb.an_w), P(rb.an_b), P(rb.qkv_w), P(rb.qkv_b), P(rb.op_w), r.a.grad, o.grad,
                           nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, pl->scale ? pl->scale + 1 : nullptr, H * W, rb.cout, o.gs, kGnEps};
      const int ids[6] = {rb.an_w, rb.an_b, rb.qkv_w, rb.qkv_b, rb.op_w, rb.op_b};
      for (int i = 0; i < 6; ++i) b.goffs[i] = G(ids[i]);
      push(b);
      ginit[o.gid] = 1;
    }
    const Tens* src[2] = {&r.x, r.has_skip ? &r.skip : nullptr};
    const int nsrc = r.has_skip ? 2 : 1;
    // ---- conv2 (+ fused projection): gradient operand of o
    gprep(o.grad, rb.cout, H, W, 0, pl->gyA);
    colsum(o.grad, pix, rb.cout, rb.cout, rb.c2.b_idx, rb.has_proj ? rb.proj.b_idx : -1);
    replay(r.in2);
    wgrad(rb.c2, pl->gyA, r.in2.n0, round_up(rb.cout, 16), rb.cout, 0, H, W);
    dgrad(rb.c2, 0, pl->gyA, H, W, pl->tA, false);
    // ---- norm2 + SiLU
    norm_bwd(r.t, pl->tA, 1, &rb.n2, 0, rb.cout, 0, 0, pl->tB, nullptr, false);
    // ---- conv1
    gprep(pl->tB, rb.cout, H, W, 0, pl->gyB);
    colsum(pl->tB, pix, rb.cout, rb.cout, rb.c1.b_idx);
    replay(r.in1);
    for (int k = 0; k < nsrc; ++k) {
      const uint8_t* act = k == 0 ? r.in1.n0 : r.in1.n1;
      wgrad(rb.c1, pl->gyB, act, round_up(src[k]->C, 16), src[k]->C, rb.c1.srcOff[k], H, W);
      float* ga = k == 0 ? pl->tA : pl->tC;
      dgrad(rb.c1, k, pl->gyB, H, W, ga, false);
      // ---- norm1 + SiLU ; the identity residual (no projection) rides along as the addend of source 0
      const float* addend = (!rb.has_proj && k == 0) ? o.grad : nullptr;
      const bool acc = was_init(*src[k]);
      norm_bwd(*src[k], ga, 1, &rb.n1, rb.c1.srcOff[k], rb.cin, 0, 0, src[k]->grad, addend, acc);
    }
    if (rb.has_proj) {  // r = proj(cat(x, skip)) (blocks.py:142): 1x1 on the raw operand
      for (int k = 0; k < nsrc; ++k) {
        const uint8_t* raw = k == 0 ? r.in1.r0 : r.in1.r1;
        wgrad(rb.proj, pl->gyA, raw, round_up(src[k]->C, 16), src[k]->C, rb.proj.srcOff[k], H, W);
        dgrad(rb.proj, k, pl->gyA, H, W, src[k]->grad, true);
      }
    }
  }

  // records [0, end) of the tape, in reverse
  int walk(int end) {
    const int B = pl->B;
    for (int i = end - 1; i >= 0; --i) {
      const Rec& r = pl->tape[i];
      if (r.kind == R_RES) {
        resblock(r);
      } else if (r.kind == R_UP) {   // Upsample (blocks.py:103-110): nearest x2 then conv
        const ConvW& cw = *r.cw;
        const int H = r.o.H, W = r.o.W;
        gprep(r.o.grad, cw.Cout, H, W, 0, pl->gyA);
        colsum(r.o.grad, (long long)B * H * W, cw.Cout, cw.Cout, cw.b_idx);
        replay(r.in1);
        wgrad(cw, pl->gyA, r.in1.n0, round_up(r.x.C, 16), r.x.C, 0, H, W);
        dgrad(cw, 0, pl->gyA, H, W, pl->tA, false);
        BOp b; b.kind = B_POOL; b.src = pl->tA; b.dst = r.x.grad; b.H = r.x.H; b.W = r.x.W; b.C = r.x.C; b.acc = was_init(r.x) ? 1 : 0;
        push(b);
      } else if (r.kind == R_DOWN) {  // Downsample (blocks.py:93-100): stride-2 conv == stride-1 conv sampled at even pixels
        const ConvW& cw = *r.cw;
        const int H = r.x.H, W = r.x.W;
        gprep(r.o.grad, cw.Cout, r.o.H, r.o.W, 2, pl->gyA);
        colsum(r.o.grad, (long long)B * r.o.H * r.o.W, cw.Cout, cw.Cout, cw.b_idx);
        replay(r.in1);
        wgrad(cw, pl->gyA, r.in1.n0, round_up(r.x.C, 16), r.x.C, 0, H, W);
        dgrad(cw, 0, pl->gyA, H, W, r.x.grad, was_init(r.x));
      } else if (r.kind == R_CONVIN) {  // weight / bias gradients only (the network input needs none)
        const ConvW& cw = *r.cw;
        const int H = r.o.H, W = r.o.W;
        gprep(r.o.grad, cw.Cout, H, W, 0, pl->gyA);
        colsum(r.o.grad, (long long)B * H * W, cw.Cout, cw.Cout, cw.b_idx);
        replay(r.in1);
        wgrad(cw, pl->gyA, r.in1.n0, cw.c0_store, cw.c0_real, 0, H, W);
        if (err) return fail("backward plan: conv_in weight gradient over %d input channels (%d after padding to 16) cannot be built: %s",
                             cw.c0_real, cw.c0_store, g_err.c_str());
      } else {
        return fail("backward plan: record %d of kind %d belongs to a model's own head", i, r.kind);
      }
      if (err) return 1;
    }
    return 0;
  }

  // C (+)= alpha * op(A) op(B); c_goff >= 0: C is that slice of the gradient buffer
  void sgemm(const float* A, long long sam, long long sak, const float* Bm, long long sbk, long long sbn, float* C, long long c_goff,
             long long ldc, int M, int N, int K, int use_inv, int acc) {
    if (c_goff >= 0 && !acc) { err = fail("backward plan: a product into the gradient buffer must add to it"); return; }
    BOp b; b.kind = B_SGEMM; b.ga = A; b.sam = sam; b.sak = sak; b.gb = Bm; b.sbk = sbk; b.sbn = sbn; b.gc = C; b.c_goff = c_goff; b.ldc = ldc;
    b.M = M; b.N = N; b.K = K; b.use_inv = use_inv; b.acc = acc; push(b);
  }
  // FiLM linears (blocks.py:39): their weight / bias gradients, then dcond = dfilm Wf, the gradient of their common input
  void film_tail() {
    const int B = pl->B, CC = core->cond_channels, R = core->film_rows;
    { BOp b; b.kind = B_FILMW; push(b); }
    const float* Wf = core->packed ? (const float*)(core->packed + core->film_w_off) : nullptr;
    sgemm(pl->dfilm, R, 1, Wf, CC, 1, pl->dcond, -1, CC, B, CC, R, 0, 0);                       // dcond = dfilm Wf
    // K = R (7168 rows for the default net) over a handful of 64 x 64 output tiles: split K across the SMs, partials in
    // pl->film_part (make_train_plan chose the split count and the buffer)
    if (pl->film_splits > 1) { pl->bops.back().chunks = pl->film_splits; pl->bops.back().part = pl->film_part; }
  }
  // nn.Embedding gradient of table `idx` from de [B][CC] (T embeddings of CC / T channels per row, actions pl->t_act [B][T])
  void embedding(const float* de, int idx, int T, int num_actions) {
    BOp b; b.kind = B_EMB; b.src = de; b.goff = G(idx); b.C = core->cond_channels; b.emb_T = T; b.emb_actions = num_actions; push(b);
  }
};

// Denoiser backward op list: conv_out(silu(norm_out(x))) (inner_model.py:48), the U-Net, then the conditioning path
// (inner_model.py:45): FiLM linears, cond_proj MLP, action embedding
int build_denoiser_bwd(const dmd_denoiser* h, BwdBuilder& bw) {
  Plan* pl = bw.pl;
  const int B = pl->B;
  bw.begin();
  {   // the last record: gF is the scaled gradient of the model output, NHWC x gF_ch channels
    const Rec& r = pl->tape.back();
    if (r.kind != R_OUT) return fail("denoiser backward plan: the tape does not end with the output head");
    const ConvW& cw = *r.cw;
    const int H = r.x.H, W = r.x.W;
    bw.gprep(pl->gF, pl->gF_ch, H, W, 0, pl->gyA);
    bw.colsum(pl->gF, (long long)B * H * W, pl->gF_ch, cw.Cout, cw.b_idx);
    bw.replay(r.in1);
    bw.wgrad(cw, pl->gyA, r.in1.n0, round_up(r.x.C, 16), r.x.C, 0, H, W);
    bw.dgrad(cw, 0, pl->gyA, H, W, pl->tA, false);
    bw.norm_bwd(r.x, pl->tA, 2, nullptr, 0, r.x.C, h->i_normout_w, h->i_normout_b, r.x.grad, nullptr, bw.was_init(r.x));
    if (bw.err) return 1;
  }
  if (bw.walk((int)pl->tape.size() - 1)) return 1;
  bw.film_tail();
  const int CC = h->cfg.cond_channels;
  const long long* goff = h->core.goff.data();
  bw.sgemm(pl->dcond, 1, CC, pl->chid, CC, 1, nullptr, goff[h->i_cp2w], CC, CC, CC, B, 1, 1);  // dW2 += dcond^T h
  bw.colsum(pl->dcond, B, CC, CC, h->i_cp2b);
  bw.sgemm(pl->dcond, CC, 1, bw.P(h->i_cp2w), CC, 1, pl->dh, -1, CC, B, CC, CC, 0, 0);          // dh = dcond W2
  { BOp b; b.kind = B_LINEAR; b.lin_in = pl->cemb; b.lin_w = bw.P(h->i_cp0w); b.lin_b = bw.P(h->i_cp0b); b.lin_out = pl->cpre; b.lin_K = CC; b.lin_F = CC; bw.push(b); }
  { BOp b; b.kind = B_DSILU; b.src = pl->cpre; b.ga = pl->dh; b.dst = pl->dpre; b.rows = (long long)B * CC; bw.push(b); }
  bw.sgemm(pl->dpre, 1, CC, pl->cemb, CC, 1, nullptr, goff[h->i_cp0w], CC, CC, CC, B, 1, 1);   // dW0 += dpre^T e
  bw.colsum(pl->dpre, B, CC, CC, h->i_cp0b);
  bw.sgemm(pl->dpre, CC, 1, bw.P(h->i_cp0w), CC, 1, pl->de, -1, CC, B, CC, CC, 0, 0);           // de = dpre W0
  bw.embedding(pl->de, h->i_actemb, h->cfg.num_steps_conditioning, h->cfg.num_actions);
  return bw.err;
}

// training workspace = forward plan (with gradient buffers) + backward temporaries.  fwd builds the forward plan (taking
// the model's own training buffers from pb.bump); bwd emits the backward op list.  cmax: the widest channel count of the
// network; gF_ch: channels of the NHWC output-gradient buffer gF (0: none).
using FwdPlanFn = std::function<int(PlanBuilder&)>;
using BwdPlanFn = std::function<int(BwdBuilder&)>;
int make_train_plan(const ModelCore& core, int cmax, int gF_ch, Plan* pl, int B, int H, int W, int T, uint8_t* base, size_t* total,
                    const FwdPlanFn& fwd, const BwdPlanFn& bwd) {
  const bool det = core.det;
  pl->train = true; pl->n_grad_tensors = 0; pl->tape.clear(); pl->det = det;
  pl->B = B; pl->H = H; pl->W = W; pl->T = T; pl->ops.clear(); pl->bops.clear();
  Bump b0{nullptr}, s0{nullptr};
  { Plan tmp; tmp.train = true; tmp.det = det; tmp.B = B; tmp.H = H; tmp.W = W; tmp.T = T; PlanBuilder pb{&core, &tmp, &b0, &s0}; if (fwd(pb)) return 1; }
  const size_t stats_bytes = (s0.off + 255) & ~(size_t)255;
  Bump sb{base}, bb{base ? base + stats_bytes : nullptr};
  if (base) { pl->base = base; pl->stats = (double*)base; pl->stats_bytes = stats_bytes; }
  if (base) { PlanBuilder pb{&core, pl, &bb, &sb}; if (fwd(pb)) return 1; } else bb.off = b0.off;
  // backward temporaries
  pl->tmp_floats = (long long)B * H * W * cmax;
  // the split attention backward at C = 128, and at every C in deterministic mode (BwdBuilder::attn_split), keeps six
  // [B][64][C] buffers in tB and four in tC
  if ((cmax > 64 || det) && pl->tmp_floats < 6ll * B * kAttnL * cmax) pl->tmp_floats = 6ll * B * kAttnL * cmax;
  const size_t act_bytes = (size_t)pl->tmp_floats * 4;
  pl->tA = (float*)bb.take(act_bytes); pl->tB = (float*)bb.take(act_bytes); pl->tC = (float*)bb.take(act_bytes);
  const size_t op_bytes = plc16_bytes(B, H, W, cmax);
  pl->gyA = (uint8_t*)bb.take(op_bytes); pl->gyB = (uint8_t*)bb.take(op_bytes);
  pl->gF = (float*)bb.take((size_t)B * H * W * gF_ch * 4); pl->gF_ch = gF_ch;
  if (init_kernels()) return 1;
  pl->partial_bytes = wgrad_partial_bytes(g_num_sms);
  pl->partial = (float*)bb.take(pl->partial_bytes);
  const int CC = core.cond_channels;
  pl->dcond = (float*)bb.take((size_t)B * CC * 4); pl->dh = (float*)bb.take((size_t)B * CC * 4); pl->cpre = (float*)bb.take((size_t)B * CC * 4);
  pl->dpre = (float*)bb.take((size_t)B * CC * 4); pl->de = (float*)bb.take((size_t)B * CC * 4);
  {   // dcond = dfilm Wf: its partials live in tA, which caps the split count at what it holds, down to kMinFilmSplits; a
      // wider cond whose partials tA cannot hold that many of keeps the full split count in a buffer of its own
    const int want = film_splits(core.film_rows);
    const long long fit = pl->tmp_floats / ((long long)B * CC);
    pl->film_part_own = 0;
    if (want <= fit || fit >= kMinFilmSplits) {
      pl->film_splits = want <= fit ? want : (int)fit;
      pl->film_part = pl->tA;
    } else {
      pl->film_splits = want;
      pl->film_part_own = splitk_partial_floats(B, CC, core.film_rows, want);
      pl->film_part = (float*)bb.take((size_t)pl->film_part_own * 4);
    }
  }
  pl->scale = (float*)bb.take(256);
  // zeroed at the start of every backward: dfilm, affine-norm sums, amax
  uint8_t* z0 = (uint8_t*)bb.take(0);
  pl->dfilm = (float*)bb.take((size_t)B * core.film_rows * 4);
  pl->nsum = (float*)bb.take((size_t)2 * B * kMaxCin * 4);
  pl->amax = (unsigned int*)bb.take(256);
  pl->zero_begin = z0; pl->zero_bytes = base ? (size_t)((uint8_t*)pl->amax + 256 - z0) : 0;
  if (total) *total = stats_bytes + bb.off + 512;
  if (!base) return 0;
  pl->bytes = stats_bytes + bb.off;
  BwdBuilder bw{&core, pl};
  if (bwd(bw)) return 1;
  pl->film_woff = (const long long*)(core.packed + core.film_woff_off); pl->film_boff = (const long long*)(core.packed + core.film_boff_off);
  return 0;
}

// U-Net / encoder level widths the executors build: GroupNorm groups of 32, and at most kMaxCin channels per operand source
// (wider convs run K-split)
bool level_width_ok(int c) { return c == 32 || c == 64 || c == 128; }
template <class Cfg> int widest_channels(const Cfg& c) {  // at least 16
  int cmax = 16;
  for (int i = 0; i < c.num_levels; ++i) cmax = c.channels[i] > cmax ? c.channels[i] : cmax;
  return cmax;
}
int make_denoiser_train_plan(const dmd_denoiser* h, Plan* pl, int B, int H, int W, uint8_t* base, size_t* total) {
  // gF: one channel per output channel, padded to 8 (the gradient-operand prep reads multiples of 8)
  return make_train_plan(h->core, widest_channels(h->cfg), round_up(h->cfg.img_channels, 8), pl, B, H, W, 1, base, total,
                         [h](PlanBuilder& pb) { return pb.build(h); }, [h](BwdBuilder& bw) { return build_denoiser_bwd(h, bw); });
}

// cond_k >= 0: the conditioning of this evaluation was computed up front by sampler_conditioning (FiLM rows at film_all + k)
// u8 != null: the frame stack is read from uint8 frames (obs is not used)
int run_forward(dmd_denoiser* h, Plan& pl, const float* noisy, const float* sigma, int sigma_is_scalar, const float* obs,
                const int64_t* act, cudaStream_t st, int prescaled = 0, StackView sv = StackView{}, int cond_k = -1,
                const U8Frames* u8 = nullptr) {
  const dmd_denoiser_config& c = h->cfg;
  const int HW = pl.H * pl.W;
  DMD_CUDA(cudaMemsetAsync(pl.stats, 0, pl.stats_bytes, st));
  const dim3 grid((HW + 255) / 256, pl.B);
  const int Cobs = c.num_steps_conditioning * c.img_channels;
  if (u8)
    pack_denoiser_input_kernel<<<grid, 256, 0, st>>>(noisy, *u8, sigma, sigma_is_scalar, pl.xin, pl.cs, Cobs, c.img_channels,
                                                     pl.CP_in, HW, c.sigma_data, c.sigma_offset_noise, prescaled, sv);
  else
    pack_denoiser_input_kernel<<<grid, 256, 0, st>>>(noisy, obs, sigma, sigma_is_scalar, pl.xin, pl.cs, Cobs, c.img_channels,
                                                     pl.CP_in, HW, c.sigma_data, c.sigma_offset_noise, prescaled, sv);
  DMD_LAUNCH_OK();
  const float* film = pl.film;
  if (cond_k >= 0) {
    film = pl.film_all + (size_t)cond_k * pl.B * h->core.film_rows;
  } else {
    const int total = pl.B * c.cond_channels;
    cond_embed_kernel<<<(total + 255) / 256, 256, 0, st>>>(pl.cs, nullptr, c.sigma_data, c.sigma_offset_noise, act, h->core.ptrs[h->i_fourier],
                                                           h->core.ptrs[h->i_actemb], pl.cemb, pl.B, pl.B, c.cond_channels, c.num_steps_conditioning,
                                                           c.num_actions, sv);
    DMD_LAUNCH_OK();
    if (linear_launch(pl.cemb, h->core.ptrs[h->i_cp0w], h->core.ptrs[h->i_cp0b], pl.chid, pl.B, c.cond_channels, c.cond_channels, 1, st)) return 1;
    if (linear_launch(pl.chid, h->core.ptrs[h->i_cp2w], h->core.ptrs[h->i_cp2b], pl.cond, pl.B, c.cond_channels, c.cond_channels, 0, st)) return 1;
    if (linear_launch(pl.cond, (const float*)(h->core.packed + h->core.film_w_off), (const float*)(h->core.packed + h->core.film_b_off), pl.film,
                      pl.B, c.cond_channels, h->core.film_rows, 0, st)) return 1;
  }
  for (const Op& op : pl.ops) {
    if (op.kind == OP_CONV) { if (conv_launch(op.conv, op.smem, op.cols, st)) return 1; }
    else if (op.kind == OP_PREP) {
      if (op.prep.film != nullptr && op.prep.film != film) { PrepParams pp = op.prep; pp.film = film; if (prep_launch(pp, op.prep_nsrc, st)) return 1; }
      else if (prep_launch(op.prep, op.prep_nsrc, st)) return 1;
    }
    else if (op.kind == OP_RESIZE) { if (resize_launch(op.rs, st, pl.det)) return 1; }
    else if (op.kind == OP_STATS) { if (gn_stats_launch(op.gn.x, op.gn.stats, pl.B, op.gn.HW, op.gn.C, op.gn.gs, pl.det, st)) return 1; }
    else { if (attn_launch(op.attn, pl.B, st)) return 1; }
  }
  return 0;
}

int run_wrap(dmd_denoiser* h, Plan& pl, const float* x, float* model_out, float* denoised, float* x_out, float* d_out,
             const float* d_prev, const float* x0, int mode, float sigma_hat, float dt, cudaStream_t st) {
  const int HW = pl.H * pl.W, total = pl.B * h->cfg.img_channels * HW;
  wrap_update_kernel<<<(total + 255) / 256, 256, 0, st>>>(pl.fout, x, pl.cs, model_out, denoised, x_out, d_out, d_prev, x0,
                                                         mode, sigma_hat, dt, h->cfg.img_channels, pl.CF, HW, total, kt_slot("wrap", (total + 255) / 256, mode));
  DMD_LAUNCH_OK();
  return 0;
}

int ensure_plan(dmd_denoiser* h, int B, int H, int W, void* ws, size_t ws_bytes) {
  DMD_CHECK(h->core.ready(), "denoiser: call dmd_denoiser_set_weights first");
  Plan& pl = h->plan;
  if (pl.B == B && pl.H == H && pl.W == W && pl.base == (uint8_t*)ws && pl.det == h->core.det) return 0;
  // size and validate on a scratch plan: the cached plan is replaced only after every check has passed, and is
  // invalidated (never left half-written) if the real build fails
  size_t need = 0;
  { Plan tmp; if (make_plan(h, &tmp, B, H, W, nullptr, &need)) return 1; }
  DMD_CHECK(ws && ws_bytes >= need, "denoiser: workspace too small (%zu < %zu)", ws_bytes, need);
  DMD_CHECK(((uintptr_t)ws & 255) == 0, "denoiser: workspace must be 256-byte aligned");
  for (auto& g : h->graphs) g.valid = false;
  if (make_plan(h, &pl, B, H, W, (uint8_t*)ws, nullptr)) { pl.B = 0; pl.base = nullptr; pl.ops.clear(); return 1; }
  return 0;
}

}  // namespace

extern "C" dmd_denoiser* dmd_denoiser_create(const dmd_denoiser_config* cfg) {
  if (!cfg || cfg->num_levels < 1 || cfg->num_levels > DMD_MAX_LEVELS) { fail("denoiser_create: bad config"); return nullptr; }
  if (cfg->num_steps_conditioning <= 0 || cfg->cond_channels <= 0 || cfg->cond_channels % 32 || cfg->cond_channels > kMaxCondChannels ||
      cfg->cond_channels % cfg->num_steps_conditioning) {
    fail("denoiser_create: cond_channels must be a multiple of 32 and of num_steps_conditioning (%d), at most %d; got %d",
         cfg->num_steps_conditioning, kMaxCondChannels, cfg->cond_channels);
    return nullptr;
  }
  for (int i = 0; i < cfg->num_levels; ++i)
    if (!level_width_ok(cfg->channels[i])) { fail("denoiser_create: channels must be 32, 64 or 128 per level, at most 128 (got %d at level %d)", cfg->channels[i], i); return nullptr; }
  {   // conv_in's operand: 16, 32 or 64 channels after padding (the operand prep and the wgrad kernel; at 128 the forward
      // computes a wrong model output)
    const int cin = (cfg->num_steps_conditioning + 1) * cfg->img_channels, cp = round_up(cin, 16);
    if (cfg->img_channels < 1 || (cp != 16 && cp != 32 && cp != 64)) {
      fail("denoiser_create: conv_in over (num_steps_conditioning + 1) * img_channels = %d input channels (%d after padding to 16) "
           "is not supported: it takes 16, 32 or 64", cin, cp);
      return nullptr;
    }
  }
  if (init_kernels()) return nullptr;
  dmd_denoiser* h = new dmd_denoiser();
  h->cfg = *cfg;
  if (build_structure(h)) { delete h; return nullptr; }
  return h;
}
extern "C" void dmd_denoiser_destroy(dmd_denoiser* h) {
  if (!h) return;
  for (auto& g : h->graphs) if (g.exec) cudaGraphExecDestroy(g.exec);
  if (h->cap_stream) cudaStreamDestroy(h->cap_stream);
  delete h;
}
extern "C" int dmd_denoiser_num_tensors(const dmd_denoiser* h) { return h->core.n_tensors; }
extern "C" size_t dmd_denoiser_packed_bytes(const dmd_denoiser* h) { return h->core.packed_bytes; }

static int pack_one(const ModelCore& m, const ConvW& c, cudaStream_t st) {
  const float* w = m.ptrs[c.w_idx];
  for (int j = 0; j < c.nchunks; ++j) {   // stored channel i of a chunk is real channel ci_off + i (c0_store = 0, c0_real = ci_off)
    const ConvChunk& ch = c.chunk[j];
    const int ci_off = (ch.src ? c.c0_real : 0) + ch.c_off;
    if (dmd_pack_conv_weight(w, m.packed + ch.pk_off, c.Cout, c.CoutPad, c.CinReal, ch.C, c.taps, ci_off, 0, c.precise, st)) return 1;
    if (c.three_pass && dmd_pack_conv_weight(w, m.packed + ch.pk_lo_off, c.Cout, c.CoutPad, c.CinReal, ch.C, c.taps, ci_off, 0, 2, st)) return 1;
  }
  if (!c.nchunks && dmd_pack_conv_weight(w, m.packed + c.pk_off, c.Cout, c.CoutPad, c.CinReal, c.Cin, c.taps, c.c0_real, c.c0_store, c.precise, st)) return 1;
  if (!c.nchunks && c.three_pass && dmd_pack_conv_weight(w, m.packed + c.pk_lo_off, c.Cout, c.CoutPad, c.CinReal, c.Cin, c.taps, c.c0_real, c.c0_store, 2, st)) return 1;
  for (int k = 0; k < c.nsrcT; ++k) {  // backward-data packs (transposed, flipped), one per concat source (and gradient chunk)
    if (!c.widthT) { if (dmd_pack_conv_weight_dgrad(w, m.packed + c.pkT_off[k], c.Cout, c.CinReal, c.srcOff[k], c.srcC[k], c.taps, st)) return 1; continue; }
    for (int j = 0; j * c.widthT < c.CoutPad; ++j) {   // output channels [j * widthT, ...) of the weight: its rows are outermost
      const int co0 = j * c.widthT, n = c.Cout - co0 < c.widthT ? c.Cout - co0 : c.widthT;
      if (dmd_pack_conv_weight_dgrad(w + (size_t)co0 * c.CinReal * c.taps, m.packed + c.pkTc_off[k][j], n, c.CinReal, c.srcOff[k], c.srcC[k],
                                     c.taps, st)) return 1;
    }
  }
  return 0;
}
static int pack_rb(const ModelCore& m, const ResBlockW& r, cudaStream_t st) {
  const int CC = m.cond_channels;
  if (r.has_proj && pack_one(m, r.proj, st)) return 1;
  if (pack_one(m, r.c1, st) || pack_one(m, r.c2, st)) return 1;
  for (const FilmW* f : {&r.n1, &r.n2}) {
    DMD_CUDA(cudaMemcpyAsync(m.packed + m.film_w_off + (size_t)f->off * CC * 4, m.ptrs[f->w_idx], (size_t)2 * f->C * CC * 4, cudaMemcpyDeviceToDevice, st));
    DMD_CUDA(cudaMemcpyAsync(m.packed + m.film_b_off + (size_t)f->off * 4, m.ptrs[f->b_idx], (size_t)2 * f->C * 4, cudaMemcpyDeviceToDevice, st));
  }
  return 0;
}

static int pack_denoiser(const dmd_denoiser* h, cudaStream_t st) {
  const ModelCore& m = h->core;
  if (pack_one(m, h->conv_in, st) || pack_one(m, h->conv_out, st)) return 1;
  for (auto& lv : h->d_blocks) for (auto& r : lv) if (pack_rb(m, r, st)) return 1;
  for (auto& lv : h->u_blocks) for (auto& r : lv) if (pack_rb(m, r, st)) return 1;
  for (auto& r : h->mid) if (pack_rb(m, r, st)) return 1;
  for (int i = 1; i < h->cfg.num_levels; ++i) if (pack_one(m, h->downs[i], st) || pack_one(m, h->ups[i], st)) return 1;
  return 0;
}

// A CUDA graph the caller captures (torch.compile's cudagraphs) replays without the host-side check that re-packs changed
// weights: the inference entry points therefore enqueue the packs as the first captured work whenever `st` is capturing, and
// every replay packs the fp32 parameters as they are then.  Inside a capture set_weights only adopts the tensors; the FiLM
// offset tables (a pageable host->device copy) must already be on the device from an uncaptured call into the same buffer.
static int stream_capturing(cudaStream_t st, bool* on) {
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  DMD_CUDA(cudaStreamIsCapturing(st, &cap));
  *on = cap != cudaStreamCaptureStatusNone;
  return 0;
}
static int set_weights_tail(ModelCore& m, cudaStream_t st, bool* pack_now) {
  bool cap = false;
  if (stream_capturing(st, &cap)) return 1;
  DMD_CHECK(!cap || m.film_rows == 0 || m.film_offsets_at == m.packed,
            "set_weights: the first call with a packed buffer cannot be captured (its FiLM offset tables are a host upload)");
  *pack_now = !cap;
  return cap ? 0 : m.upload_film_offsets(st);
}

extern "C" int dmd_denoiser_set_weights(dmd_denoiser* h, const float* const* ptrs_host, int n_ptrs, void* packed, void* stream) {
  DMD_CHECK(h, "set_weights: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  bool moved = false, pack_now = false;
  if (h->core.set_weights("InnerModel", ptrs_host, n_ptrs, packed, &moved)) return 1;
  if (moved) { h->plan.B = 0; h->core.tplans.clear(); for (auto& g : h->graphs) g.valid = false; }
  if (set_weights_tail(h->core, st, &pack_now)) return 1;
  return pack_now ? pack_denoiser(h, st) : 0;
}

// deterministic mode: plans, sampler graphs and workspace queries made while it is on use the fixed-order arms
extern "C" int dmd_denoiser_set_deterministic(dmd_denoiser* h, int on) {
  DMD_CHECK(h, "denoiser_set_deterministic: null handle");
  h->core.det = on != 0;
  return 0;
}
extern "C" int dmd_rew_end_set_deterministic(dmd_rew_end* h, int on) {
  DMD_CHECK(h, "rew_end_set_deterministic: null handle");
  h->core.det = on != 0;
  return 0;
}

extern "C" size_t dmd_denoiser_workspace_bytes(const dmd_denoiser* h, int B, int H, int W) {
  Plan tmp; size_t need = 0;
  if (make_plan(h, &tmp, B, H, W, nullptr, &need)) return 0;
  return need;
}

extern "C" int dmd_denoiser_forward(dmd_denoiser* h, int B, int H, int W, const float* noisy, const float* sigma,
                                    int sigma_is_scalar, const float* obs, const int64_t* act, float* out_model,
                                    float* out_denoised, void* workspace, size_t workspace_bytes, void* stream) {
  DMD_CHECK(h && noisy && sigma && obs && act, "denoiser_forward: null argument");
  if (ensure_plan(h, B, H, W, workspace, workspace_bytes)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  if (run_forward(h, h->plan, noisy, sigma, sigma_is_scalar, obs, act, st)) return 1;
  return run_wrap(h, h->plan, noisy, out_model, out_denoised, nullptr, nullptr, nullptr, nullptr, 0, 1.f, 0.f, st);
}

extern "C" int dmd_inner_model_forward(dmd_denoiser* h, int B, int H, int W, const float* noisy_rescaled,
                                       const float* c_noise, int c_noise_is_scalar, const float* obs_rescaled,
                                       const int64_t* act, float* out, void* workspace, size_t workspace_bytes,
                                       void* stream) {
  DMD_CHECK(h && noisy_rescaled && c_noise && obs_rescaled && act && out, "inner_model_forward: null argument");
  if (ensure_plan(h, B, H, W, workspace, workspace_bytes)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  if (run_forward(h, h->plan, noisy_rescaled, c_noise, c_noise_is_scalar, obs_rescaled, act, st, 1)) return 1;
  return run_wrap(h, h->plan, noisy_rescaled, out, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 1.f, 0.f, st);
}

// the arguments the two uint8 InnerModel entry points share, each named in its message
static int inner_model_u8_args(const char* who, const dmd_denoiser* h, const float* noisy_rescaled, const float* c_noise,
                               const dmd_u8_frames* obs, const int64_t* act, const float* out, U8Frames* u8) {
  DMD_CHECK(h, "%s: handle is NULL", who);
  DMD_CHECK(noisy_rescaled, "%s: noisy_rescaled is NULL", who);
  DMD_CHECK(c_noise, "%s: c_noise is NULL", who);
  DMD_CHECK(act, "%s: act is NULL", who);
  DMD_CHECK(out, "%s: out is NULL", who);
  return u8_frames_arg(who, "obs", obs, u8);
}

extern "C" int dmd_inner_model_forward_u8(dmd_denoiser* h, int B, int H, int W, const float* noisy_rescaled, const float* c_noise,
                                          int c_noise_is_scalar, const dmd_u8_frames* obs, const int64_t* act, float* out,
                                          void* workspace, size_t workspace_bytes, void* stream) {
  U8Frames u8;
  if (inner_model_u8_args("inner_model_forward_u8", h, noisy_rescaled, c_noise, obs, act, out, &u8)) return 1;
  if (ensure_plan(h, B, H, W, workspace, workspace_bytes)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  if (run_forward(h, h->plan, noisy_rescaled, c_noise, c_noise_is_scalar, nullptr, act, st, 1, StackView{}, -1, &u8)) return 1;
  return run_wrap(h, h->plan, noisy_rescaled, out, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 1.f, 0.f, st);
}

// ---------------------------------------------------------------------------------------------- training entry points
namespace {

// any_mode: a backward finds the plan its forward ran on (one per workspace) in whichever mode that forward was planned
Plan* find_train_plan(ModelCore& core, int B, int H, int W, int T, const void* ws, bool any_mode = false) {
  for (auto& p : core.tplans)
    if (p->B == B && p->H == H && p->W == W && p->T == T && p->base == (const uint8_t*)ws && (any_mode || p->det == core.det)) return p.get();
  return nullptr;
}

// make(pl, base, total): make_train_plan of the model; who: the model's name in messages
using MakeTrainPlanFn = std::function<int(Plan*, uint8_t*, size_t*)>;
int ensure_train_plan(ModelCore& core, const char* who, int B, int H, int W, int T, void* ws, size_t ws_bytes,
                      const MakeTrainPlanFn& make, Plan** out) {
  DMD_CHECK(core.ready(), "%s: call dmd_%s_set_weights first", who, who);
  if ((*out = find_train_plan(core, B, H, W, T, ws)) != nullptr) return 0;
  size_t need = 0;
  { Plan tmp; if (make(&tmp, nullptr, &need)) return 1; }
  DMD_CHECK(ws && ws_bytes >= need, "%s: training workspace too small (%zu < %zu)", who, ws_bytes, need);
  DMD_CHECK(((uintptr_t)ws & 255) == 0, "%s: workspace must be 256-byte aligned", who);
  // a plan bound to the same workspace with another shape is stale; keep at most 8 plans
  auto& tp = core.tplans;
  for (size_t i = 0; i < tp.size();)
    if (tp[i]->base == (uint8_t*)ws) tp.erase(tp.begin() + i); else ++i;
  if (tp.size() >= 8) tp.erase(tp.begin());
  std::unique_ptr<Plan> pl(new Plan());
  if (make(pl.get(), (uint8_t*)ws, nullptr)) return 1;
  *out = pl.get();
  tp.push_back(std::move(pl));
  return 0;
}

// start of every backward: the accumulators of the plan (dfilm, affine-norm sums, amax) cleared, and the caller's flat gradient
// buffer too unless the call adds to it (the *_backward_accumulate entry points)
int clear_backward(const ModelCore& core, Plan& pl, float* grads, int accumulate, cudaStream_t st) {
  if (!accumulate) DMD_CUDA(cudaMemsetAsync(grads, 0, (size_t)core.grad_total * 4, st));
  DMD_CUDA(cudaMemsetAsync(pl.zero_begin, 0, pl.zero_bytes, st));
  return 0;
}

// one op of a backward op list; inv: the reciprocal of the loss scale (device scalar) the parameter gradients are multiplied by
int run_bop(const ModelCore& core, const Plan& pl, const BOp& b, float* grads, const float* inv, cudaStream_t st) {
  const int B = pl.B;
  switch (b.kind) {
    case B_PREP: if (prep_launch(b.prep, b.prep_nsrc, st)) return 1; break;
    case B_CONV: if (conv_launch(b.conv, b.smem, b.cols, st)) return 1; break;
    case B_WGRAD: if (wgrad_launch(b.wg, grads + b.goff, st)) return 1; break;
    case B_COLSUM:
      if (colsum_launch(b.src, grads + b.goff, b.goff2 >= 0 ? grads + b.goff2 : nullptr, inv, b.rows, b.C, b.Creal, st,
                        pl.det ? pl.partial : nullptr, pl.partial_bytes)) return 1;
      break;
    case B_NORM1: if (norm_bwd_launch(b.nb, 1, st, pl.det)) return 1; break;
    case B_NORM2: if (norm_bwd_launch(b.nb, 2, st)) return 1; break;
    case B_AFFINE: if (affine_param_grad_launch(b.nb, grads + b.goff, grads + b.goff2, inv, st)) return 1; break;
    case B_POOL: if (sumpool2_launch(b.src, b.dst, B, b.H, b.W, b.C, b.acc, st)) return 1; break;
    case B_ATTN: {
      AttnBwdParams ab = b.ab;
      ab.dgamma = grads + b.goffs[0]; ab.dbeta = grads + b.goffs[1]; ab.dwqkv = grads + b.goffs[2]; ab.dbqkv = grads + b.goffs[3];
      ab.dwout = grads + b.goffs[4]; ab.dbout = grads + b.goffs[5];
      if (attn_bwd_launch(ab, B, st)) return 1;
      break;
    }
    case B_ATTN_RECOMP: {
      const dim3 grid((b.ap.L + kAttnTile - 1) / kAttnTile, B);
      if (b.ap.C == 128) attn_qkv_kernel<128><<<grid, kAttnQkvThreads, 0, st>>>(b.ap);
      else if (b.ap.C == 64) attn_qkv_kernel<64><<<grid, kAttnQkvThreads, 0, st>>>(b.ap);
      else attn_qkv_kernel<32><<<grid, kAttnQkvThreads, 0, st>>>(b.ap);
      DMD_LAUNCH_OK();
      const long long total = (long long)B * b.ap.L * b.ap.C;
      attn_xn_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(b.ap.x, b.ap.st_in, b.ap.gamma, b.ap.beta, b.at_xn, b.ap.L, b.ap.C,
                                                                     b.ap.gs, b.ap.eps, total);
      DMD_LAUNCH_OK();
      break;
    }
    case B_ATTN_CORE:
      if (b.ap.L == kAttnL)
        attn_core_bwd_kernel<kAttnL><<<dim3(b.ap.C / 8, B), kAttnCoreThreads, 0, st>>>(b.ap.scratch, b.at_gy, b.ap.out, b.at_y, b.at_gqkv,
                                                                                      b.at_gxn, b.ap.C, b.ap.L);
      else
        attn_core_bwd_kernel<0><<<dim3(b.ap.C / 8, B), kAttnCoreThreads, 0, st>>>(b.ap.scratch, b.at_gy, b.ap.out, b.at_y, b.at_gqkv,
                                                                                 b.at_gxn, b.ap.C, b.ap.L);
      DMD_LAUNCH_OK();
      break;
    case B_MEMSET: DMD_CUDA(cudaMemsetAsync(b.ms_ptr, 0, b.ms_bytes, st)); break;
    case B_SGEMM:   // the long-K products are split: dcond = dfilm Wf (K = all FiLM rows, partials in film_part) and the
                    // attention weight gradients (K = every token of the batch, partials in tA)
      if (sgemm_launch(b.ga, b.sam, b.sak, b.gb, b.sbk, b.sbn, b.c_goff >= 0 ? grads + b.c_goff : b.gc, b.ldc, b.M, b.N, b.K,
                       b.use_inv ? inv : nullptr, b.acc, b.chunks, b.part ? b.part : pl.tA, st)) return 1;
      break;
    case B_FILMW:
      if (film_wgrad_launch(pl.dfilm, pl.cond, grads, pl.film_woff, pl.film_boff, B, core.film_rows, core.cond_channels, inv, st)) return 1;
      break;
    case B_LINEAR: if (linear_launch(b.lin_in, b.lin_w, b.lin_b, b.lin_out, B, b.lin_K, b.lin_F, 0, st)) return 1; break;
    case B_DSILU: if (dsilu_mul_launch(b.src, b.ga, b.dst, b.rows, st)) return 1; break;
    case B_EMB:
      if (embedding_bwd_launch(b.src, pl.t_act, grads + b.goff, B, b.C, b.emb_T, b.emb_actions, inv, st, pl.det)) return 1;
      break;
    default: return fail("backward: unknown op kind %d", b.kind);
  }
  return 0;
}
// the backward op list; the caller has cleared (clear_backward), set the loss scale and seeded the gradient the list starts from.
// Every op that writes into `grads` ADDS to it (wgrad reduce with accumulate = 1, colsum / attention / embedding atomics, affine
// and FiLM +=, sgemm into a c_goff slice with acc = 1, checked when the list is built), so an accumulating call is this same list
// on a buffer that was not cleared
int run_backward(const ModelCore& core, Plan& pl, float* grads, cudaStream_t st) {
  for (const BOp& b : pl.bops)
    if (run_bop(core, pl, b, grads, pl.scale + 1, st)) return 1;
  return 0;
}

}  // namespace

// ---- per-op entry point of the split attention backward: BwdBuilder::attn_split's op list on a one-block model, run by
// run_bop.  Workspace: the backward temporaries tA / tB / tC at the size attn_split needs (6 x B x L x C floats each; a
// training plan's are at least that large, and split_k's split count is min(K / 256, 32) either way for C <= 128), the
// deterministic column sums' partials and the norm backward's per-channel sums.
static size_t attn_split_workspace(int B, int L, int C, uint8_t* base, Plan* pl) {
  Bump bb{base};
  const long long tmp = 6ll * B * L * C;
  float* t[3];
  for (float*& p : t) p = (float*)bb.take((size_t)tmp * 4);
  const size_t part = std::max(colsum_partial_bytes((long long)B * L, C), colsum_partial_bytes((long long)B * L, 3 * C));
  float* partial = (float*)bb.take(part);
  float* nsum = (float*)bb.take((size_t)2 * B * kMaxCin * 4);
  if (pl) {
    pl->B = B; pl->tmp_floats = tmp; pl->tA = t[0]; pl->tB = t[1]; pl->tC = t[2];
    pl->partial = partial; pl->partial_bytes = part; pl->nsum = nsum;
  }
  return bb.off;
}
extern "C" size_t dmd_attn_split_bwd_workspace_bytes(int B, int L, int C) {
  return B > 0 && L > 0 && C > 0 ? attn_split_workspace(B, L, C, nullptr, nullptr) : 0;
}
extern "C" int dmd_attn_split_bwd(const float* x, const double* stats_in, const float* gamma, const float* beta, const float* wqkv,
                                  const float* bqkv, const float* wout, const float* gout, float* gx, float* grads,
                                  const long long* goffs, const float* inv_scale, int B, int L, int C, int gs, int det,
                                  void* workspace, size_t workspace_bytes, void* stream) {
  DMD_CHECK(x && stats_in && gamma && beta && wqkv && bqkv && wout && gout && gx && grads && goffs && workspace,
            "attn_split_bwd: null argument");
  DMD_CHECK((C == 32 || C == 64 || C == 128) && L >= 1 && L <= kAttnL && B >= 1 && B <= 65535,
            "attn_split_bwd: unsupported shape B=%d L=%d C=%d (C in {32, 64, 128}, 1 <= L <= %d)", B, L, C, kAttnL);
  DMD_CHECK(gs > 0 && gs % 8 == 0 && C % gs == 0 && C / gs <= 8, "attn_split_bwd: bad group size %d for C=%d", gs, C);
  for (int i = 0; i < 6; ++i) DMD_CHECK(goffs[i] >= 0, "attn_split_bwd: gradient offset %d is negative", i);
  DMD_CHECK(((uintptr_t)workspace & 255) == 0, "attn_split_bwd: workspace must be 256-byte aligned");
  DMD_CHECK(workspace_bytes >= attn_split_workspace(B, L, C, nullptr, nullptr), "attn_split_bwd: workspace too small (%zu < %zu)",
            workspace_bytes, attn_split_workspace(B, L, C, nullptr, nullptr));
  if (init_kernels()) return 1;
  // gamma, beta, Wqkv, bqkv, Wout, bout: state_dict tensors 0..5 of the one-block model (bout's value is not read)
  ModelCore core;
  core.ptrs = {gamma, beta, wqkv, bqkv, wout, nullptr};
  core.goff.assign(goffs, goffs + 6);
  core.n_tensors = 6;
  ResBlockW rb{};
  rb.cin = rb.cout = C; rb.has_attn = 1;
  rb.an_w = 0; rb.an_b = 1; rb.qkv_w = 2; rb.qkv_b = 3; rb.op_w = 4; rb.op_b = 5;
  Tens o{const_cast<float*>(x), const_cast<double*>(stats_in), C, 1, L, gs};
  o.grad = gx;
  Plan pl;
  pl.det = det != 0;
  attn_split_workspace(B, L, C, (uint8_t*)workspace, &pl);
  BwdBuilder bw{&core, &pl};
  bw.begin();
  bw.attn_split(rb, o, gout);
  if (bw.err) return 1;
  for (const BOp& b : pl.bops)
    if (run_bop(core, pl, b, grads, inv_scale, (cudaStream_t)stream)) return 1;
  return 0;
}

// ---- per-layer entry points of one nn.Conv2d: the ConvW of Walker::conv on a one-conv model, packed by pack_one and launched
// through the executors' own expansions (for_each_conv_launch, for_each_dgrad_launch, for_each_wgrad_launch).  The *_plan
// twins run the same expansions on stand-in pointers and record what they emit, without a device.
struct dmd_conv_layer { ModelCore core; ConvW cw; };

extern "C" dmd_conv_layer* dmd_conv_layer_create(int cout, int cin_real, int taps, int c0_real, int c0_store, int c1, int split, int dgrad) {
  // the walker itself refuses a conv that needs more than kMaxConvChunks K-split or backward-data chunks
  if (!(cout > 0 && cout <= 128 && (taps == 1 || taps == 9) && c0_real > 0 && c0_real <= c0_store && c0_store % 16 == 0 && c1 >= 0 &&
        c1 % 16 == 0 && cin_real == c0_real + c1)) {
    fail("conv_layer: unsupported conv %d -> %d (taps %d, first source %d real in %d stored, second source %d)", cin_real, cout, taps,
         c0_real, c0_store, c1);
    return nullptr;
  }
  std::unique_ptr<dmd_conv_layer> h(new dmd_conv_layer());
  Walker w{&h->core};
  h->cw = w.conv(cout, cin_real, taps, c0_real, c0_store, c1, split != 0, dgrad != 0);
  if (w.err) return nullptr;   // dmd_last_error() says why
  h->core.finish(w.pk);
  return h.release();
}
extern "C" void dmd_conv_layer_destroy(dmd_conv_layer* h) { delete h; }

namespace {

// the one-launch description of the layer's forward, as PlanBuilder::conv and the actor-critic's run_conv fill it: the caller's
// operands, bias, residual, output and statistics, the layer's weights and split-fp16 mode.  plane: bytes of one PLC16 plane
int layer_fprop_desc(const dmd_conv_layer* h, const uint8_t* packed, const dmd_conv_desc* d, dmd_conv_desc* o, size_t* plane) {
  DMD_CHECK(h && packed && d && d->src0 && d->out, "conv_layer: null layer, packed buffer, descriptor, src0 or out");
  const ConvW& cw = h->cw;
  DMD_CHECK(d->C0 == cw.c0_store && d->C1 == cw.Cin - cw.c0_store, "conv_layer: operand channels %d+%d, the layer takes %d+%d", d->C0,
            d->C1, cw.c0_store, cw.Cin - cw.c0_store);
  const bool split = cw.precise || cw.three_pass;
  if (split) DMD_CHECK(d->src0_lo && (!d->C1 || d->src1_lo), "conv_layer: a split-fp16 layer needs the low operand parts");
  DMD_CHECK(!d->wpk_x, "conv_layer: a layer carries no fused projection");
  DMD_CHECK(d->B > 0 && d->H > 0 && d->W > 0, "conv_layer: bad size %dx%dx%d", d->B, d->H, d->W);
  *o = *d;
  if (!split) o->src0_lo = o->src1_lo = nullptr;
  o->wpk = packed + cw.pk_off; o->precise = cw.precise; o->taps = cw.taps; o->Cout = cw.Cout; o->CoutPad = cw.CoutPad;
  *plane = (size_t)plc_geometry(d->B, d->H, d->W).Qalloc * 16;   // one PLC16 plane holds 8 channels
  return 0;
}

int layer_wgrad_check(const dmd_conv_layer* h, int Ca, int Cin, int ci_off) {
  DMD_CHECK(h, "conv_layer: null layer");
  DMD_CHECK(Cin > 0 && Cin <= Ca && ci_off >= 0 && ci_off + Cin <= h->cw.CinReal, "conv_layer_wgrad: input channels [%d, %d + %d) of %d (Ca %d)",
            ci_off, ci_off, Cin, h->cw.CinReal, Ca);
  return 0;
}

// stand-in pointers of the host-only twins, far apart so that each pointer an expansion emits names the operand it points into
// (0 src0 / gradient, 1 src1 / activation, 2 src0_lo, 3 src1_lo, 4 residual, 5 out, 6 bias, 7 statistics, 8 packed buffer)
constexpr uintptr_t kTwinSpan = 1ull << 40;
inline uint8_t* twin(int i) { return (uint8_t*)(kTwinSpan * (uintptr_t)(i + 1)); }
void twin_locate(const void* p, size_t plane, int* which, long long* at) {
  if (!p) { *which = -1; *at = 0; return; }
  const uintptr_t u = (uintptr_t)p, off = u % kTwinSpan;
  *which = (int)(u / kTwinSpan) - 1;
  *at = off % plane ? -1 : (long long)(off / plane);
}
struct TwinRecorder {
  dmd_conv_layer_launch* out; int cap; int n = 0;
  dmd_conv_layer_launch* next() {
    if (n >= cap) { fail("conv_layer plan: more than %d launches", cap); return nullptr; }
    dmd_conv_layer_launch* L = out + n++;
    memset(L, 0, sizeof(*L));
    return L;
  }
  int conv(const dmd_conv_desc& x, size_t plane) {
    ConvParams p; size_t smem; int cols;
    if (conv_fill(&x, &p, &smem, &cols)) return 1;   // the launch's own checks, as dmd_conv_plan runs them
    dmd_conv_layer_launch* L = next();
    if (!L) return 1;
    const void* srcs[4] = {x.src0, x.src1, x.src0_lo, x.src1_lo};
    for (int i = 0; i < 4; ++i) twin_locate(srcs[i], plane, &L->src[i], &L->plane[i]);
    L->C0 = x.C0; L->C1 = x.C1; L->precise = x.precise;
    L->wpk = (long long)((const uint8_t*)x.wpk - twin(8));
    L->bias = x.bias != nullptr; L->residual = x.residual && x.residual != x.out; L->residual_is_out = x.residual && x.residual == x.out;
    L->stats = x.out_stats != nullptr;
    L->Cout = x.Cout; L->CoutPad = x.CoutPad;
    return 0;
  }
  int wgrad(const WgradLaunch& W, size_t plane) {
    dmd_conv_layer_launch* L = next();
    if (!L) return 1;
    twin_locate(W.wp.a_plane[0], plane, &L->src[0], &L->plane[0]);
    twin_locate(W.wp.b_plane[0], plane, &L->src[1], &L->plane[1]);
    L->src[2] = L->src[3] = -1;
    for (int j = 0; j < 8; ++j) L->Cg += W.wp.a_plane[j] ? 8 : 0;
    L->C0 = W.rp.N;
    L->co_off = W.rp.co_off; L->ci_off = W.rp.ci_off; L->Cout = W.rp.Cout; L->Cin = W.rp.Cin;
    return 0;
  }
};

int layer_fprop_twin(const dmd_conv_layer* h, const dmd_conv_desc* d, dmd_conv_layer_launch* out, int cap, int* n) {
  DMD_CHECK(d && out && n, "conv_layer plan: null argument");
  dmd_conv_desc s = *d;   // the caller's pointers say only which operands are present
  const void** ps[8] = {&s.src0, &s.src1, &s.src0_lo, &s.src1_lo, (const void**)&s.residual, (const void**)&s.out, (const void**)&s.bias,
                        (const void**)&s.out_stats};
  for (int i = 0; i < 8; ++i) if (*ps[i]) *ps[i] = twin(i);
  dmd_conv_desc dc; size_t plane;
  if (layer_fprop_desc(h, twin(8), &s, &dc, &plane)) return 1;
  TwinRecorder r{out, cap};
  if (for_each_conv_launch(h->cw, dc, plane, [&](size_t off) { return twin(8) + off; },
                           [&](const dmd_conv_desc& x) { return r.conv(x, plane); })) return 1;
  *n = r.n;
  return 0;
}
int layer_dgrad_twin(const dmd_conv_layer* h, int k, int B, int H, int W, int accumulate, dmd_conv_layer_launch* out, int cap, int* n) {
  DMD_CHECK(h && out && n, "conv_layer plan: null argument");
  DMD_CHECK(k >= 0 && k < h->cw.nsrcT, "conv_layer_dgrad: source %d has no backward-data pack (the layer has %d)", k, h->cw.nsrcT);
  DMD_CHECK(B > 0 && H > 0 && W > 0, "conv_layer_dgrad: bad size %dx%dx%d", B, H, W);
  const size_t plane = (size_t)plc_geometry(B, H, W).Qalloc * 16;
  TwinRecorder r{out, cap};
  if (for_each_dgrad_launch(h->cw, k, twin(8), twin(0), B, H, W, (float*)twin(5), accumulate != 0,
                            [&](const dmd_conv_desc& x) { return r.conv(x, plane); })) return 1;
  *n = r.n;
  return 0;
}
int layer_wgrad_twin(const dmd_conv_layer* h, int Ca, int Cin, int ci_off, int B, int H, int W, dmd_conv_layer_launch* out, int cap, int* n) {
  DMD_CHECK(out && n, "conv_layer plan: null argument");
  if (layer_wgrad_check(h, Ca, Cin, ci_off)) return 1;
  DMD_CHECK(B > 0 && H > 0 && W > 0, "conv_layer_wgrad: bad size %dx%dx%d", B, H, W);
  const size_t plane = (size_t)plc_geometry(B, H, W).Qalloc * 16;
  TwinRecorder r{out, cap};
  if (for_each_wgrad_launch(h->cw, twin(0), twin(1), Ca, Cin, ci_off, B, H, W, (float*)twin(7), nullptr,
                            [&](const WgradLaunch& L) { return r.wgrad(L, plane); })) return 1;
  *n = r.n;
  return 0;
}

}  // namespace

extern "C" int dmd_conv_layer_info(const dmd_conv_layer* h, dmd_conv_layer_shape* out) {
  DMD_CHECK(h && out, "conv_layer_info: null argument");
  const ConvW& cw = h->cw;
  memset(out, 0, sizeof(*out));
  out->Cin = cw.Cin; out->CoutPad = cw.CoutPad; out->nchunks = cw.nchunks; out->precise = cw.precise; out->three_pass = cw.three_pass;
  out->widthT = cw.widthT; out->nsrcT = cw.nsrcT; out->packed_bytes = h->core.packed_bytes;
  // launch counts at an 8 x 8 image, with both sources (and their low parts) present
  dmd_conv_layer_launch L[3 * kMaxConvChunks];
  const int cap = 3 * kMaxConvChunks, c1 = cw.Cin - cw.c0_store;
  dmd_conv_desc d; memset(&d, 0, sizeof(d));
  d.src0 = d.src0_lo = d.out = (float*)1; d.src1 = d.src1_lo = c1 ? (const void*)1 : nullptr;
  d.C0 = cw.c0_store; d.C1 = c1; d.B = 1; d.H = d.W = 8; d.stride = 1;
  if (layer_fprop_twin(h, &d, L, cap, &out->fprop_launches)) return 1;
  for (int k = 0; k < cw.nsrcT; ++k)
    if (layer_dgrad_twin(h, k, 1, 8, 8, 0, L, cap, &out->dgrad_launches[k])) return 1;
  const int ca[2] = {cw.c0_store, c1}, cin[2] = {cw.c0_real, c1};
  for (int k = 0; k < (c1 ? 2 : 1); ++k)
    if (layer_wgrad_twin(h, ca[k], cin[k], k ? cw.c0_real : 0, 1, 8, 8, L, cap, &out->wgrad_launches[k])) return 1;
  return 0;
}
extern "C" int dmd_conv_layer_fprop_plan(const dmd_conv_layer* h, const dmd_conv_desc* d, dmd_conv_layer_launch* out, int cap, int* n) {
  return layer_fprop_twin(h, d, out, cap, n);
}
extern "C" int dmd_conv_layer_dgrad_plan(const dmd_conv_layer* h, int k, int B, int H, int W, int accumulate, dmd_conv_layer_launch* out,
                                         int cap, int* n) {
  return layer_dgrad_twin(h, k, B, H, W, accumulate, out, cap, n);
}
extern "C" int dmd_conv_layer_wgrad_plan(const dmd_conv_layer* h, int Ca, int Cin, int ci_off, int B, int H, int W,
                                         dmd_conv_layer_launch* out, int cap, int* n) {
  return layer_wgrad_twin(h, Ca, Cin, ci_off, B, H, W, out, cap, n);
}

extern "C" int dmd_conv_layer_pack(const dmd_conv_layer* h, const float* w, void* packed, void* stream) {
  DMD_CHECK(h && w && packed, "conv_layer_pack: null argument");
  DMD_CHECK(((uintptr_t)packed & 255) == 0, "conv_layer_pack: the packed buffer must be 256-byte aligned");
  ModelCore m;   // the layer's weight (tensor 0) and packed buffer
  m.ptrs = {w, nullptr};
  m.packed = (uint8_t*)packed;
  return pack_one(m, h->cw, (cudaStream_t)stream);
}
extern "C" int dmd_conv_layer_fprop(const dmd_conv_layer* h, const void* packed, const dmd_conv_desc* d, void* stream) {
  dmd_conv_desc dc; size_t plane;
  if (layer_fprop_desc(h, (const uint8_t*)packed, d, &dc, &plane)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  return for_each_conv_launch(h->cw, dc, plane, [&](size_t off) { return (const uint8_t*)packed + off; },
                              [&](const dmd_conv_desc& x) { return dmd_conv2d_fprop(&x, st); });
}
extern "C" int dmd_conv_layer_dgrad(const dmd_conv_layer* h, const void* packed, int k, const void* gy, int B, int H, int W, float* out,
                                    int accumulate, void* stream) {
  DMD_CHECK(h && packed && gy && out, "conv_layer_dgrad: null argument");
  DMD_CHECK(k >= 0 && k < h->cw.nsrcT, "conv_layer_dgrad: source %d has no backward-data pack (the layer has %d)", k, h->cw.nsrcT);
  cudaStream_t st = (cudaStream_t)stream;
  return for_each_dgrad_launch(h->cw, k, (const uint8_t*)packed, (const uint8_t*)gy, B, H, W, out, accumulate != 0,
                               [&](const dmd_conv_desc& x) { return dmd_conv2d_fprop(&x, st); });
}
extern "C" int dmd_conv_layer_wgrad(const dmd_conv_layer* h, const void* gy, const void* act, int Ca, int Cin, int ci_off, int B, int H,
                                    int W, void* partial, size_t partial_bytes, const float* inv_scale, float* dW, void* stream) {
  DMD_CHECK(gy && act && partial && dW, "conv_layer_wgrad: null argument");
  if (layer_wgrad_check(h, Ca, Cin, ci_off)) return 1;
  if (init_kernels()) return 1;
  DMD_CHECK(partial_bytes >= wgrad_partial_bytes(g_num_sms), "conv_layer_wgrad: partial buffer too small (%zu < %zu)", partial_bytes,
            wgrad_partial_bytes(g_num_sms));
  cudaStream_t st = (cudaStream_t)stream;
  return for_each_wgrad_launch(h->cw, (const uint8_t*)gy, (const uint8_t*)act, Ca, Cin, ci_off, B, H, W, (float*)partial, inv_scale,
                               [&](const WgradLaunch& L) { return wgrad_launch(L, dW, st); });
}

extern "C" size_t dmd_denoiser_train_workspace_bytes(const dmd_denoiser* h, int B, int H, int W) {
  Plan tmp; size_t need = 0;
  if (make_denoiser_train_plan(h, &tmp, B, H, W, nullptr, &need)) return 0;
  return need;
}
extern "C" int dmd_denoiser_train_dcond_plan(const dmd_denoiser* h, int B, int H, int W, int* splits, long long* own_partial_floats,
                                             long long* temporary_floats) {
  DMD_CHECK(splits && own_partial_floats && temporary_floats, "denoiser_train_dcond_plan: null output");
  Plan tmp; size_t need = 0;
  if (make_denoiser_train_plan(h, &tmp, B, H, W, nullptr, &need)) return 1;
  *splits = tmp.film_splits; *own_partial_floats = tmp.film_part_own; *temporary_floats = tmp.tmp_floats;
  return 0;
}
extern "C" long long dmd_denoiser_grad_layout(const dmd_denoiser* h, long long* offsets, long long* numels, int n) {
  return grad_layout(h ? &h->core : nullptr, offsets, numels, n);
}

extern "C" int dmd_inner_model_forward_train(dmd_denoiser* h, int B, int H, int W, const float* noisy_rescaled, const float* c_noise,
                                             int c_noise_is_scalar, const float* obs_rescaled, const int64_t* act, float* out,
                                             void* workspace, size_t workspace_bytes, void* stream) {
  DMD_CHECK(h && noisy_rescaled && c_noise && obs_rescaled && act && out, "inner_model_forward_train: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  Plan* pl = nullptr;
  auto make = [h, B, H, W](Plan* p, uint8_t* base, size_t* total) { return make_denoiser_train_plan(h, p, B, H, W, base, total); };
  if (ensure_train_plan(h->core, "denoiser", B, H, W, 1, workspace, workspace_bytes, make, &pl)) return 1;
  pl->t_act = act;
  if (run_forward(h, *pl, noisy_rescaled, c_noise, c_noise_is_scalar, obs_rescaled, act, st, 1)) return 1;
  return run_wrap(h, *pl, noisy_rescaled, out, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 1.f, 0.f, st);
}

extern "C" int dmd_inner_model_forward_train_u8(dmd_denoiser* h, int B, int H, int W, const float* noisy_rescaled, const float* c_noise,
                                                int c_noise_is_scalar, const dmd_u8_frames* obs, const int64_t* act, float* out,
                                                void* workspace, size_t workspace_bytes, void* stream) {
  U8Frames u8;
  if (inner_model_u8_args("inner_model_forward_train_u8", h, noisy_rescaled, c_noise, obs, act, out, &u8)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  Plan* pl = nullptr;
  auto make = [h, B, H, W](Plan* p, uint8_t* base, size_t* total) { return make_denoiser_train_plan(h, p, B, H, W, base, total); };
  if (ensure_train_plan(h->core, "denoiser", B, H, W, 1, workspace, workspace_bytes, make, &pl)) return 1;
  pl->t_act = act;
  if (run_forward(h, *pl, noisy_rescaled, c_noise, c_noise_is_scalar, nullptr, act, st, 1, StackView{}, -1, &u8)) return 1;
  return run_wrap(h, *pl, noisy_rescaled, out, nullptr, nullptr, nullptr, nullptr, nullptr, 0, 1.f, 0.f, st);
}

static int denoiser_backward_impl(const char* who, dmd_denoiser* h, int B, int H, int W, const float* grad_out, float* grads,
                                  long long grads_numel, int accumulate, void* workspace, void* stream) {
  DMD_CHECK(h && grad_out && grads && workspace, "%s: null argument", who);
  Plan* plp = find_train_plan(h->core, B, H, W, 1, workspace, true);
  DMD_CHECK(plp && plp->train, "%s: no matching dmd_inner_model_forward_train on this workspace (B=%d H=%d W=%d)", who, B, H, W);
  Plan& pl = *plp;
  DMD_CHECK(grads_numel >= h->core.grad_total, "%s: gradient buffer too small (%lld < %lld floats)", who, grads_numel, h->core.grad_total);
  DMD_CHECK(((uintptr_t)grads & 15) == 0, "%s: gradient buffer must be 16-byte aligned", who);
  cudaStream_t st = (cudaStream_t)stream;
  const int HW = H * W, C = h->cfg.img_channels;
  if (clear_backward(h->core, pl, grads, accumulate, st)) return 1;
  // loss scale from the incoming gradient, then the scaled NHWC gradient of the model output
  if (loss_scale_launch(grad_out, (long long)B * C * HW, pl.amax, pl.scale, st)) return 1;
  nchw_to_nhwc_scaled_kernel<<<dim3((HW + 255) / 256, B), 256, 0, st>>>(grad_out, pl.gF, pl.scale, C, pl.gF_ch, HW);
  DMD_LAUNCH_OK();
  return run_backward(h->core, pl, grads, st);
}
extern "C" int dmd_denoiser_backward(dmd_denoiser* h, int B, int H, int W, const float* grad_out, float* grads, long long grads_numel,
                                     void* workspace, void* stream) {
  return denoiser_backward_impl("denoiser_backward", h, B, H, W, grad_out, grads, grads_numel, 0, workspace, stream);
}
extern "C" int dmd_denoiser_backward_accumulate(dmd_denoiser* h, int B, int H, int W, const float* grad_out, float* grads,
                                                long long grads_numel, void* workspace, void* stream) {
  return denoiser_backward_impl("denoiser_backward_accumulate", h, B, H, W, grad_out, grads, grads_numel, 1, workspace, stream);
}

// ---------------------------------------------------------------------------------------------- sampler
namespace {

__global__ void fill_scalar_kernel(float* p, float v) { *p = v; }
struct SigmaList { float v[kMaxSamplerEvals]; };
__global__ void write_sigmas_kernel(float* dst, SigmaList s, int n) { if ((int)threadIdx.x < n) dst[threadIdx.x] = s.v[threadIdx.x]; }

struct SamplerIO { const float* obs; const int64_t* act; StackView sv; float* traj; const float* eps; float* out; };

// DiffusionSampler.sample (diffusion_sampler.py:31-58).  traj[0] holds x ~ N(0, 1) on entry; traj[i+1] receives the iterate after
// step i (the reference's `trajectory` list); the last iterate additionally goes to io.out when that is not the last
// trajectory slot (e.g. straight into the WorldModelEnv's frame ring).  No staging copies: every buffer is used in place.
int sampler_body(dmd_denoiser* h, const dmd_sampler_config* sc, const SamplerIO& io, cudaStream_t st) {
  Plan& pl = h->plan;
  const dmd_denoiser_config& c = h->cfg;
  const int n = sc->num_sigmas;
  const size_t img_elems = (size_t)pl.B * c.img_channels * pl.H * pl.W;
  const int total = (int)img_elems;
  // diffusion_sampler.py:35  gamma_ = min(s_churn / (len(sigmas) - 1), 2**0.5 - 1)
  const double gamma_ = std::fmin((double)sc->s_churn / (double)(n - 1), std::sqrt(2.0) - 1.0);
  // ---- the sigma of every U-Net evaluation is host-known: conditioning (Fourier + action embedding -> cond MLP -> all 44 FiLM
  //      linears) of ALL evaluations in four launches up front instead of four per evaluation inside the loop
  SigmaList sl; int K = 0; bool hoist = true;
  for (int i = 0; i + 1 < n && hoist; ++i) {
    const float sigma = sc->sigmas_host[i], next_sigma = sc->sigmas_host[i + 1];
    if (K + 2 > kMaxSamplerEvals) { hoist = false; break; }
    sl.v[K++] = sigma;   // the network is conditioned on sigma, NOT sigma_hat (diffusion_sampler.py:44)
    if (!(sc->order == 1 || next_sigma == 0.0f)) sl.v[K++] = next_sigma;
  }
  float* sig_dev = pl.cs + (size_t)pl.B * 4;  // spare slot after cs: the un-hoisted fallback's scalar sigma
  if (hoist) {
    write_sigmas_kernel<<<1, 32, 0, st>>>(pl.sig_all, sl, K);
    DMD_LAUNCH_OK();
    const int rows = K * pl.B, CC = c.cond_channels;
    cond_embed_kernel<<<(rows * CC + 255) / 256, 256, 0, st>>>(nullptr, pl.sig_all, c.sigma_data, c.sigma_offset_noise, io.act, h->core.ptrs[h->i_fourier],
                                                               h->core.ptrs[h->i_actemb], pl.cemb_all, rows, pl.B, CC, c.num_steps_conditioning, c.num_actions, io.sv);
    DMD_LAUNCH_OK();
    if (linear_launch(pl.cemb_all, h->core.ptrs[h->i_cp0w], h->core.ptrs[h->i_cp0b], pl.chid_all, rows, CC, CC, 1, st)) return 1;
    if (linear_launch(pl.chid_all, h->core.ptrs[h->i_cp2w], h->core.ptrs[h->i_cp2b], pl.cond_all, rows, CC, CC, 0, st)) return 1;
    if (linear_launch(pl.cond_all, (const float*)(h->core.packed + h->core.film_w_off), (const float*)(h->core.packed + h->core.film_b_off), pl.film_all,
                      rows, CC, h->core.film_rows, 0, st)) return 1;
  }
  int k = 0;
  auto forward = [&](const float* x, float sigma_value) -> int {
    if (hoist) { const int kk = k++; return run_forward(h, pl, x, pl.sig_all + kk, 1, io.obs, io.act, st, 0, io.sv, kk); }
    fill_scalar_kernel<<<1, 1, 0, st>>>(sig_dev, sigma_value);
    DMD_LAUNCH_OK();
    return run_forward(h, pl, x, sig_dev, 1, io.obs, io.act, st, 0, io.sv, -1);
  };
  for (int i = 0; i + 1 < n; ++i) {
    const float sigma = sc->sigmas_host[i], next_sigma = sc->sigmas_host[i + 1];
    const double gamma = (sc->s_tmin <= sigma && sigma <= sc->s_tmax) ? gamma_ : 0.0;
    const float sigma_hat = sigma * (float)(gamma + 1.0);
    const float* x = io.traj + (size_t)i * img_elems;
    float* xn = io.traj + (size_t)(i + 1) * img_elems;
    if (gamma > 0.0) {  // churn: x + eps * sqrt(sigma_hat^2 - sigma^2) (diffusion_sampler.py:41-43); the trajectory keeps the un-churned x
      DMD_CHECK(io.eps != nullptr, "sampler: s_churn > 0 needs eps noise from the caller");
      DMD_CHECK(sc->s_noise == 1.0f, "sampler: s_noise != 1 not built yet");
      const float cfac = std::sqrt(sigma_hat * sigma_hat - sigma * sigma);
      axpy_kernel<<<(total + 255) / 256, 256, 0, st>>>(x, io.eps + (size_t)i * img_elems, cfac, pl.s_xc, total);
      DMD_LAUNCH_OK();
      x = pl.s_xc;
    }
    if (forward(x, sigma)) return 1;
    const float dt = next_sigma - sigma_hat;
    if (sc->order == 1 || next_sigma == 0.0f) {
      if (run_wrap(h, pl, x, nullptr, nullptr, xn, nullptr, nullptr, nullptr, 1, sigma_hat, dt, st)) return 1;
    } else {
      // Heun: x_2 = x + d*dt ; denoise(x_2, next_sigma) ; x = x + ((d + d_2)/2)*dt
      if (run_wrap(h, pl, x, nullptr, nullptr, pl.s_x2, pl.s_d, nullptr, nullptr, 1, sigma_hat, dt, st)) return 1;
      if (forward(pl.s_x2, next_sigma)) return 1;
      if (run_wrap(h, pl, pl.s_x2, nullptr, nullptr, xn, nullptr, pl.s_d, x, 2, next_sigma, dt, st)) return 1;
    }
  }
  float* last = io.traj + (size_t)(n - 1) * img_elems;
  if (io.out && io.out != last) DMD_CUDA(cudaMemcpyAsync(io.out, last, img_elems * 4, cudaMemcpyDeviceToDevice, st));
  return 0;
}

}  // namespace

extern "C" int dmd_sampler_sample(dmd_denoiser* h, const dmd_sampler_config* sc, int B, int H, int W, const float* prev_obs,
                                  const int64_t* prev_act, int ring_head, float* traj, const float* eps, float* out_x,
                                  void* workspace, size_t workspace_bytes, int use_graph, void* stream) {
  DMD_CHECK(h && sc && prev_obs && prev_act && traj, "sampler: null argument");
  DMD_CHECK(sc->num_sigmas >= 2 && sc->sigmas_host, "sampler: need at least 2 sigmas");
  DMD_CHECK(sc->order == 1 || sc->order == 2, "sampler: order must be 1 or 2");
  cudaStream_t st = (cudaStream_t)stream;
  const dmd_denoiser_config& c = h->cfg;
  const int n = sc->num_sigmas, T = c.num_steps_conditioning;
  DMD_CHECK(ring_head >= -1 && ring_head < T, "sampler: ring_head must be -1 (contiguous stacks) or a slot index < %d", T);
  if (init_kernels()) return 1;
  if (h->need_B != B || h->need_H != H || h->need_W != W || h->need_det != h->core.det) {
    h->need_bytes = dmd_denoiser_workspace_bytes(h, B, H, W);
    h->need_B = B; h->need_H = H; h->need_W = W; h->need_det = h->core.det;
  }
  DMD_CHECK(h->need_bytes > 0, "sampler: %s", g_err.c_str());
  DMD_CHECK(workspace_bytes >= h->need_bytes, "sampler: workspace too small (%zu < %zu)", workspace_bytes, h->need_bytes);
  if (ensure_plan(h, B, H, W, workspace, workspace_bytes)) return 1;
  SamplerIO io; memset(&io, 0, sizeof(io));
  io.obs = prev_obs; io.act = prev_act; io.traj = traj; io.eps = eps; io.out = out_x;
  if (ring_head >= 0) {  // frames (T, B, C, H, W), acts (T, B); logical slot k = physical (ring_head + k) % T
    const long long chw = (long long)c.img_channels * H * W;
    io.sv = StackView{T, ring_head, (long long)B * chw, chw, (long long)B, 1};
  }
  bool cap = false;
  if (stream_capturing(st, &cap)) return 1;
  if (cap) return pack_denoiser(h, st) || sampler_body(h, sc, io, st);   // inside the caller's graph: no graph of our own
  if (!use_graph) return sampler_body(h, sc, io, st);

  const float churn[4] = {sc->s_churn, sc->s_tmin, sc->s_tmax, sc->s_noise};
  SamplerGraph* g = nullptr;
  for (auto& cand : h->graphs) {
    if (cand.valid && cand.B == B && cand.H == H && cand.W == W && cand.ws == workspace && cand.order == sc->order &&
        cand.obs == prev_obs && cand.act == prev_act && cand.traj == traj && cand.eps == eps && cand.out == out_x &&
        cand.sv.ring_T == io.sv.ring_T && cand.sv.head == io.sv.head && (int)cand.sigmas.size() == n &&
        memcmp(cand.sigmas.data(), sc->sigmas_host, 4 * n) == 0 && memcmp(cand.churn, churn, sizeof(churn)) == 0) { g = &cand; break; }
  }
  if (!g) {
    // graphs bake the buffer addresses in: one graph per distinct set (a WorldModelEnv cycles through T ring heads); keep 8
    if (h->graphs.size() >= 8) {
      size_t victim = 0;
      for (size_t i = 1; i < h->graphs.size(); ++i) if (h->graphs[i].stamp < h->graphs[victim].stamp) victim = i;
      if (h->graphs[victim].exec) cudaGraphExecDestroy(h->graphs[victim].exec);
      h->graphs.erase(h->graphs.begin() + victim);
    }
    SamplerGraph ng;
    cudaGraph_t graph = nullptr;
    if (!h->cap_stream) DMD_CUDA(cudaStreamCreateWithFlags(&h->cap_stream, cudaStreamNonBlocking));
    DMD_CUDA(cudaStreamBeginCapture(h->cap_stream, cudaStreamCaptureModeThreadLocal));
    const long long before = g_launches;
    int rc = sampler_body(h, sc, io, h->cap_stream);
    cudaError_t ce = cudaStreamEndCapture(h->cap_stream, &graph);
    ng.kernels = g_launches - before;
    g_launches = before;  // capture does not execute
    if (rc) { if (graph) cudaGraphDestroy(graph); return 1; }
    DMD_CHECK(ce == cudaSuccess, "sampler: graph capture failed: %s", cudaGetErrorString(ce));
    ce = cudaGraphInstantiate(&ng.exec, graph, 0);
    cudaGraphDestroy(graph);
    DMD_CHECK(ce == cudaSuccess, "sampler: graph instantiate failed: %s", cudaGetErrorString(ce));
    ng.valid = true; ng.B = B; ng.H = H; ng.W = W; ng.ws = workspace; ng.order = sc->order; ng.has_eps = eps != nullptr;
    ng.obs = prev_obs; ng.act = prev_act; ng.traj = traj; ng.eps = eps; ng.out = out_x; ng.sv = io.sv;
    ng.sigmas.assign(sc->sigmas_host, sc->sigmas_host + n); memcpy(ng.churn, churn, sizeof(churn));
    h->graphs.push_back(ng);
    g = &h->graphs.back();
  }
  g->stamp = ++h->graph_clock;
  DMD_CUDA(cudaGraphLaunch(g->exec, st));
  g_launches += g->kernels;
  return 0;
}

// ---------------------------------------------------------------------------------------------- actor-critic executor
// Immediate mode: its workspaces are pooled per autograd node (one per imagined step), so a cached plan per workspace would
// multiply host state for launches that take microseconds to describe.  Forward convs of the encoder run in split-fp16 (error
// ~2^-22): MaxPool2d (actor_critic.py:109) turns a 2^-11 operand rounding into a different arg-max in a few windows, which
// moves the encoder GRADIENTS by several per cent against the fp32 reference (measured: 2.6e-2 whole-gradient error with fp16
// operands, 1.8e-4 with an exact forward).  The encoder is 0.12 GFLOP, so the 3x tensor work is noise.
struct dmd_actor_critic {
  dmd_actor_critic_config cfg;
  ModelCore core;
  struct Level { int cin, cout, down; int gn_w, gn_b; ConvW conv; int has_skip; ConvW skip; };
  ConvW conv0;
  std::vector<Level> levels;
  int i_wih = 0, i_whh = 0, i_bih = 0, i_bhh = 0, i_cw = 0, i_cb = 0, i_aw = 0, i_ab = 0;
  int feat_c = 0, feat_hw = 0;
};

namespace {

struct AcBuffers {
  float* x0; void* opnd; void* opnd_lo; std::vector<float*> r, y, pooled; std::vector<double*> st_in, st_y; float *gates, *hx, *cx; double* stats; size_t stats_bytes; size_t total;
};

// channels of the operand and gradient buffers that every level shares: the widest level, and never fewer than the 64 the
// layouts of 32- and 64-channel nets have always had
int ac_operand_channels(const dmd_actor_critic_config& c) { const int w = widest_channels(c); return w > 64 ? w : 64; }

// lays out the workspace; base may be null (size query)
int ac_layout(const dmd_actor_critic* h, int B, uint8_t* base, AcBuffers* o) {
  const dmd_actor_critic_config& c = h->cfg;
  Bump sb{base};
  const size_t nl = h->levels.size();
  o->st_in.resize(nl + 1); o->st_y.resize(nl);
  int S = c.img_size;
  // statistics first (one memset)
  for (size_t i = 0; i <= nl; ++i) {
    const int C = i == 0 ? c.channels[0] : h->levels[i - 1].cout;
    o->st_in[i] = (double*)sb.take((size_t)B * (C / gn_group_size(C)) * 2 * 8);
  }
  o->stats = (double*)base; o->stats_bytes = (sb.off + 255) & ~(size_t)255;
  Bump bb{base ? base + o->stats_bytes : nullptr};
  o->x0 = (float*)bb.take((size_t)B * S * S * h->conv0.c0_store * 4);
  const int cw = ac_operand_channels(c);
  o->opnd = bb.take(plc16_bytes(B, S, S, cw));  // one operand buffer: every conv's prep immediately precedes it on the stream
  o->opnd_lo = bb.take(plc16_bytes(B, S, S, cw));  // its fp16 low part (split-fp16 forward)
  float* cur = (float*)bb.take((size_t)B * S * S * c.channels[0] * 4);  // conv0 output
  o->r.assign(nl, nullptr); o->y.assign(nl, nullptr); o->pooled.assign(nl + 1, nullptr);
  o->pooled[0] = cur;
  for (size_t i = 0; i < nl; ++i) {
    const auto& lv = h->levels[i];
    if (lv.has_skip) o->r[i] = (float*)bb.take((size_t)B * S * S * lv.cout * 4);
    o->y[i] = (float*)bb.take((size_t)B * S * S * lv.cout * 4);
    if (lv.down) { S /= 2; o->pooled[i + 1] = (float*)bb.take((size_t)B * S * S * lv.cout * 4); }
    else o->pooled[i + 1] = o->y[i];
  }
  o->gates = (float*)bb.take((size_t)B * 4 * c.lstm_dim * 4);
  o->total = o->stats_bytes + bb.off + 256;
  return 0;
}

}  // namespace

extern "C" dmd_actor_critic* dmd_actor_critic_create(const dmd_actor_critic_config* cfg) {
  if (!cfg || cfg->num_levels < 1 || cfg->num_levels > DMD_MAX_LEVELS) { fail("actor_critic_create: bad config"); return nullptr; }
  for (int i = 0; i < cfg->num_levels; ++i)
    if (!level_width_ok(cfg->channels[i])) { fail("actor_critic_create: channels must be 32, 64 or 128 per level, at most 128 (got %d at level %d)", cfg->channels[i], i); return nullptr; }
  if (cfg->lstm_dim % 4) { fail("actor_critic_create: lstm_dim must be a multiple of 4"); return nullptr; }
  if (init_kernels()) return nullptr;
  dmd_actor_critic* h = new dmd_actor_critic();
  h->cfg = *cfg;
  Walker w{&h->core};
  // registration order (actor_critic.py:41-47,101-110): encoder.encoder.{0: Conv3x3, k: SmallResBlock(f.0.norm, f.2, skip_projection),
  // MaxPool...}, lstm.{weight_ih, weight_hh, bias_ih, bias_hh}, critic_linear, actor_linear
  h->conv0 = w.conv(cfg->channels[0], cfg->img_channels, 9, cfg->img_channels, round_up(cfg->img_channels, 16), 0, true, false);
  int S = cfg->img_size;
  for (int i = 0; i < cfg->num_levels; ++i) {
    dmd_actor_critic::Level lv;
    lv.cin = cfg->channels[i > 0 ? i - 1 : 0]; lv.cout = cfg->channels[i]; lv.down = cfg->down[i] ? 1 : 0;
    lv.gn_w = w.next(lv.cin); lv.gn_b = w.next(lv.cin);
    lv.conv = w.conv(lv.cout, lv.cin, 9, lv.cin, lv.cin, 0, true);
    lv.has_skip = lv.cin != lv.cout;
    if (lv.has_skip) lv.skip = w.conv(lv.cout, lv.cin, 1, lv.cin, lv.cin, 0, true);
    h->levels.push_back(lv);
    if (lv.down) S /= 2;
  }
  h->feat_c = cfg->channels[cfg->num_levels - 1]; h->feat_hw = S * S;
  const long long D = cfg->lstm_dim, K = (long long)h->feat_c * h->feat_hw;
  h->i_wih = w.next(4 * D * K); h->i_whh = w.next(4 * D * D); h->i_bih = w.next(4 * D); h->i_bhh = w.next(4 * D);
  h->i_cw = w.next(D); h->i_cb = w.next(1); h->i_aw = w.next((long long)cfg->num_actions * D); h->i_ab = w.next(cfg->num_actions);
  h->core.finish(w.pk);
  if (w.err) { delete h; return nullptr; }
  return h;
}
extern "C" void dmd_actor_critic_destroy(dmd_actor_critic* h) { delete h; }
extern "C" int dmd_actor_critic_num_tensors(const dmd_actor_critic* h) { return h->core.n_tensors; }
extern "C" size_t dmd_actor_critic_packed_bytes(const dmd_actor_critic* h) { return h->core.packed_bytes; }

extern "C" int dmd_actor_critic_set_weights(dmd_actor_critic* h, const float* const* ptrs_host, int n_ptrs, void* packed, void* stream) {
  DMD_CHECK(h, "set_weights: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  bool moved = false;   // nothing is cached between calls
  if (h->core.set_weights("ActorCritic", ptrs_host, n_ptrs, packed, &moved)) return 1;
  if (pack_one(h->core, h->conv0, st)) return 1;
  for (auto& lv : h->levels) if (pack_one(h->core, lv.conv, st) || (lv.has_skip && pack_one(h->core, lv.skip, st))) return 1;
  return 0;
}

extern "C" int dmd_actor_critic_set_deterministic(dmd_actor_critic* h, int on) {
  DMD_CHECK(h, "actor_critic_set_deterministic: null handle");
  h->core.det = on != 0;
  return 0;
}
extern "C" size_t dmd_actor_critic_workspace_bytes(const dmd_actor_critic* h, int B) {
  AcBuffers b; ac_layout(h, B, nullptr, &b); return b.total;
}

extern "C" int dmd_actor_critic_forward(dmd_actor_critic* h, int B, const float* obs, const float* hx_in, const float* cx_in,
                                        float* logits, float* val, float* hx_out, float* cx_out, void* workspace,
                                        size_t workspace_bytes, void* stream) {
  DMD_CHECK(h && obs && hx_in && cx_in && logits && val && hx_out && cx_out && workspace, "ac forward: null argument");
  DMD_CHECK(h->core.ready(), "ac forward: call dmd_actor_critic_set_weights first");
  DMD_CHECK(((uintptr_t)workspace & 255) == 0, "ac forward: workspace must be 256-byte aligned");
  const dmd_actor_critic_config& c = h->cfg;
  const ModelCore& m = h->core;
  cudaStream_t st = (cudaStream_t)stream;
  AcBuffers b; ac_layout(h, B, (uint8_t*)workspace, &b);
  DMD_CHECK(workspace_bytes >= b.total, "ac forward: workspace too small (%zu < %zu)", workspace_bytes, b.total);
  const bool det = m.det;
  DMD_CUDA(cudaMemsetAsync(b.stats, 0, b.stats_bytes, st));
  int S = c.img_size;
  if (dmd_nchw_to_nhwc(obs, b.x0, B, c.img_channels, h->conv0.c0_store, S * S, st)) return 1;
  // every conv reads the hi + lo parts of one operand buffer, written by the prep just before it
  auto run_conv = [&](const ConvW& cw, const float* src, int Csrc, int hw, int mode, int gamma_idx, int beta_idx, const double* st_in,
                      const float* resid, float* out, double* st_out) -> int {
    dmd_prep_desc pd = prep_desc(src, Csrc, B, hw, hw, 0, mode, st_in, m.P(gamma_idx), m.P(beta_idx), b.opnd, b.opnd_lo);
    if (dmd_prep_act(&pd, st)) return 1;
    dmd_conv_desc d; memset(&d, 0, sizeof(d));
    d.src0 = b.opnd; d.src0_lo = b.opnd_lo; d.precise = cw.precise; d.C0 = round_up(Csrc, 16);
    d.B = B; d.H = hw; d.W = hw; d.taps = cw.taps; d.stride = 1;
    d.wpk = m.packed + cw.pk_off; d.bias = m.ptrs[cw.b_idx]; d.Cout = cw.Cout; d.CoutPad = cw.CoutPad;
    d.residual = resid; d.out = out; d.out_stats = st_out; d.out_gs = gn_group_size(cw.Cout);
    const bool stats_after = st_out && (det || !conv_epilogue_stats_fit(hw, hw));   // as PlanBuilder::conv
    if (stats_after) d.out_stats = nullptr;
    const size_t plane = (size_t)plc_geometry(B, hw, hw).Qalloc * 16;   // one PLC16 plane holds 8 channels
    if (for_each_conv_launch(cw, d, plane, [&](size_t off) { return m.packed + off; },
                             [&](const dmd_conv_desc& dc) { return dmd_conv2d_fprop(&dc, st); })) return 1;
    return stats_after ? gn_stats_launch(out, st_out, B, hw * hw, cw.Cout, d.out_gs, det, st) : 0;
  };
  // conv0 feeds the first GroupNorm -> statistics in its epilogue
  if (run_conv(h->conv0, b.x0, h->conv0.c0_store, S, 0, 0, 0, nullptr, nullptr, b.pooled[0], b.st_in[0])) return 1;
  for (size_t i = 0; i < h->levels.size(); ++i) {
    const auto& lv = h->levels[i];
    const float* x = b.pooled[i];
    const float* r = x;
    if (lv.has_skip) { if (run_conv(lv.skip, x, lv.cin, S, 0, 0, 0, nullptr, nullptr, b.r[i], nullptr)) return 1; r = b.r[i]; }
    // SmallResBlock: skip(x) + conv3x3(silu(GroupNorm(x)))  (blocks.py:122-123)
    double* st_y = lv.down ? nullptr : b.st_in[i + 1];
    if (run_conv(lv.conv, x, lv.cin, S, 2, lv.gn_w, lv.gn_b, b.st_in[i], r, b.y[i], st_y)) return 1;
    if (lv.down) {
      double* st_pool = i + 1 < h->levels.size() ? b.st_in[i + 1] : nullptr;
      if (maxpool2_stats_launch(b.y[i], b.pooled[i + 1], det ? nullptr : st_pool, B, S, S, lv.cout, gn_group_size(lv.cout), st)) return 1;
      if (det && st_pool && gn_stats_launch(b.pooled[i + 1], st_pool, B, (S / 2) * (S / 2), lv.cout, gn_group_size(lv.cout), true, st)) return 1;
      S /= 2;
    }
  }
  const float* feat = b.pooled[h->levels.size()];
  const int K = h->feat_c * h->feat_hw, D = c.lstm_dim;
  if (linear_launch(feat, m.ptrs[h->i_wih], m.ptrs[h->i_bih], b.gates, B, K, 4 * D, 0, st, 0, h->feat_hw)) return 1;
  if (linear_launch(hx_in, m.ptrs[h->i_whh], m.ptrs[h->i_bhh], b.gates, B, D, 4 * D, 0, st, 1, 0)) return 1;
  if (lstm_gates_launch(b.gates, cx_in, hx_out, cx_out, B, D, st)) return 1;
  if (linear_launch(hx_out, m.ptrs[h->i_aw], m.ptrs[h->i_ab], logits, B, D, c.num_actions, 0, st)) return 1;
  if (linear_launch(hx_out, m.ptrs[h->i_cw], m.ptrs[h->i_cb], val, B, D, 1, 0, st)) return 1;
  return 0;
}


// ---------------------------------------------------------------------------------------------- actor-critic training
// ActorCritic.predict_act_value under autograd (actor_critic.py:68-73, called with grad from env_loop.py:31,57): the forward
// above leaves every activation in its workspace; dmd_actor_critic_backward consumes it.  One call = one autograd node of
// the BPTT graph; torch's engine chains the nodes through (g_hx_in, g_cx_in) and accumulates the parameter gradients.
namespace {

struct AcScratch {
  float *g_a, *g_b, *tA; uint8_t *gy_op, *x_op; float *dgates, *g_h, *g_xflat, *x_flat, *nsum, *scale, *partial; unsigned int* amax; size_t total, partial_bytes;
};
int ac_scratch_layout(const dmd_actor_critic* h, int B, uint8_t* base, AcScratch* o) {
  const dmd_actor_critic_config& c = h->cfg;
  Bump bb{base};
  const int S = c.img_size, cw = ac_operand_channels(c);
  const size_t act = (size_t)B * S * S * cw * 4;
  o->g_a = (float*)bb.take(act); o->g_b = (float*)bb.take(act); o->tA = (float*)bb.take(act);
  o->gy_op = (uint8_t*)bb.take(plc16_bytes(B, S, S, cw)); o->x_op = (uint8_t*)bb.take(plc16_bytes(B, S, S, cw));
  const int D = c.lstm_dim, K = h->feat_c * h->feat_hw;
  o->dgates = (float*)bb.take((size_t)B * 4 * D * 4); o->g_h = (float*)bb.take((size_t)B * D * 4);
  o->g_xflat = (float*)bb.take((size_t)B * K * 4); o->x_flat = (float*)bb.take((size_t)B * K * 4);
  o->nsum = (float*)bb.take((size_t)2 * B * kMaxCin * 4);
  o->scale = (float*)bb.take(256); o->amax = (unsigned int*)bb.take(256);
  if (init_kernels()) return 1;
  o->partial_bytes = wgrad_partial_bytes(g_num_sms);
  o->partial = (float*)bb.take(o->partial_bytes);
  o->total = bb.off + 256;
  return 0;
}

}  // namespace

extern "C" size_t dmd_actor_critic_backward_scratch_bytes(const dmd_actor_critic* h, int B) {
  AcScratch s; if (ac_scratch_layout(h, B, nullptr, &s)) return 0; return s.total;
}
extern "C" long long dmd_actor_critic_grad_layout(const dmd_actor_critic* h, long long* offsets, long long* numels, int n) {
  return grad_layout(h ? &h->core : nullptr, offsets, numels, n);
}

static int ac_backward_impl(dmd_actor_critic* h, int B, const float* hx_in, const float* cx_in, const float* hx_out,
                            const float* g_logits, const float* g_val, const float* g_hx, const float* g_cx,
                            float* grads, long long grads_numel, int accumulate, float* g_hx_in, float* g_cx_in, void* workspace,
                            void* scratch, size_t scratch_bytes, void* stream);
extern "C" int dmd_actor_critic_backward(dmd_actor_critic* h, int B, const float* hx_in, const float* cx_in, const float* hx_out,
                                         const float* g_logits, const float* g_val, const float* g_hx, const float* g_cx,
                                         float* grads, long long grads_numel, float* g_hx_in, float* g_cx_in, void* workspace,
                                         void* scratch, size_t scratch_bytes, void* stream) {
  return ac_backward_impl(h, B, hx_in, cx_in, hx_out, g_logits, g_val, g_hx, g_cx, grads, grads_numel, 0, g_hx_in, g_cx_in, workspace, scratch, scratch_bytes, stream);
}
extern "C" int dmd_actor_critic_backward_accumulate(dmd_actor_critic* h, int B, const float* hx_in, const float* cx_in, const float* hx_out,
                                                    const float* g_logits, const float* g_val, const float* g_hx, const float* g_cx,
                                                    float* grads, long long grads_numel, float* g_hx_in, float* g_cx_in, void* workspace,
                                                    void* scratch, size_t scratch_bytes, void* stream) {
  return ac_backward_impl(h, B, hx_in, cx_in, hx_out, g_logits, g_val, g_hx, g_cx, grads, grads_numel, 1, g_hx_in, g_cx_in, workspace, scratch, scratch_bytes, stream);
}
// every parameter-gradient writer below ADDS its (un-scaled) contribution, so "accumulate" is simply "do not clear the buffer first"
static int ac_backward_impl(dmd_actor_critic* h, int B, const float* hx_in, const float* cx_in, const float* hx_out,
                            const float* g_logits, const float* g_val, const float* g_hx, const float* g_cx,
                            float* grads, long long grads_numel, int accumulate, float* g_hx_in, float* g_cx_in, void* workspace,
                            void* scratch, size_t scratch_bytes, void* stream) {
  DMD_CHECK(h && hx_in && cx_in && hx_out && grads && g_hx_in && g_cx_in && workspace && scratch, "ac backward: null argument");
  DMD_CHECK(h->core.ready(), "ac backward: call dmd_actor_critic_set_weights first");
  DMD_CHECK(grads_numel >= h->core.grad_total && ((uintptr_t)grads & 15) == 0, "ac backward: bad gradient buffer");
  DMD_CHECK(((uintptr_t)scratch & 255) == 0, "ac backward: scratch must be 256-byte aligned");
  const dmd_actor_critic_config& c = h->cfg;
  const ModelCore& m = h->core;
  cudaStream_t st = (cudaStream_t)stream;
  AcBuffers b; ac_layout(h, B, (uint8_t*)workspace, &b);
  AcScratch sc; if (ac_scratch_layout(h, B, (uint8_t*)scratch, &sc)) return 1;
  DMD_CHECK(scratch_bytes >= sc.total, "ac backward: scratch too small (%zu < %zu)", scratch_bytes, sc.total);
  const int D = c.lstm_dim, A = c.num_actions, K = h->feat_c * h->feat_hw;
  auto G = [&](int idx) { return grads + m.goff[idx]; };
  auto sgemm = [&](const float* Am, long long sam, long long sak, const float* Bm, long long sbk, long long sbn, float* C, long long ldc,
                   int M, int N, int Kd, int acc) -> int {
    return sgemm_launch(Am, sam, sak, Bm, sbk, sbn, C, ldc, M, N, Kd, nullptr, acc, 0, nullptr, st);
  };
  auto colsum = [&](const float* x, long long rows, int C, int Creal, float* out, float* out2, const float* inv) -> int {
    return colsum_launch(x, out, out2, inv, rows, C, Creal, st, m.det ? sc.partial : nullptr, sc.partial_bytes);
  };
  if (!accumulate) DMD_CUDA(cudaMemsetAsync(grads, 0, (size_t)m.grad_total * 4, st));
  DMD_CUDA(cudaMemsetAsync(sc.amax, 0, 256, st));
  // ---- heads (actor_critic.py:73)
  if (heads_bwd_launch(g_hx, g_logits, g_val, hx_out, m.ptrs[h->i_aw], m.ptrs[h->i_cw], sc.g_h, G(h->i_ab), G(h->i_cw), G(h->i_cb), B, D, A, st)) return 1;
  if (g_logits && sgemm(g_logits, 1, A, hx_out, D, 1, G(h->i_aw), D, A, D, B, 1)) return 1;   // dWa += g_logits^T h'
  // ---- LSTMCell (actor_critic.py:72)
  if (lstm_cell_bwd_launch(b.gates, cx_in, sc.g_h, g_cx, sc.dgates, g_cx_in, B, D, st)) return 1;
  const float* feat = b.pooled[h->levels.size()];
  if (dmd_nhwc_to_nchw(feat, sc.x_flat, B, h->feat_c, h->feat_c, h->feat_hw, st)) return 1;   // x.flatten(start_dim=1) of the NCHW feature map
  if (sgemm(sc.dgates, 1, 4 * D, sc.x_flat, K, 1, G(h->i_wih), K, 4 * D, K, B, 1)) return 1;  // dWih += dgates^T x
  if (sgemm(sc.dgates, 1, 4 * D, hx_in, D, 1, G(h->i_whh), D, 4 * D, D, B, 1)) return 1;      // dWhh += dgates^T hx
  if (colsum(sc.dgates, B, 4 * D, 4 * D, G(h->i_bih), G(h->i_bhh), nullptr)) return 1;
  if (sgemm(sc.dgates, 4 * D, 1, m.ptrs[h->i_whh], D, 1, g_hx_in, D, B, D, 4 * D, 0)) return 1;   // g_hx = dgates Whh
  if (sgemm(sc.dgates, 4 * D, 1, m.ptrs[h->i_wih], K, 1, sc.g_xflat, K, B, K, 4 * D, 0)) return 1;  // g_x = dgates Wih
  // ---- encoder (actor_critic.py:101-113): the feature gradient enters the fp16 tensor-core path with a loss scale
  float* g_cur = sc.g_a;    // gradient of pooled[i+1]; g_a / g_b ping-pong down the encoder
  auto other = [&](float* p) { return p == sc.g_a ? sc.g_b : sc.g_a; };
  if (dmd_nchw_to_nhwc(sc.g_xflat, g_cur, B, h->feat_c, h->feat_c, h->feat_hw, st)) return 1;
  {
    const long long n = (long long)B * K;
    if (loss_scale_launch(g_cur, n, sc.amax, sc.scale, st)) return 1;
    scale_inplace_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g_cur, sc.scale, n);
    DMD_LAUNCH_OK();
  }
  const float* inv = sc.scale + 1;
  auto wgrad = [&](const ConvW& cw, const uint8_t* gy, const uint8_t* act, int Ca, int hw) -> int {
    return for_each_wgrad_launch(cw, gy, act, Ca, cw.CinReal, 0, B, hw, hw, sc.partial, inv,
                                 [&](const WgradLaunch& L) { return wgrad_launch(L, G(cw.w_idx), st); });
  };
  auto dgrad = [&](const ConvW& cw, const uint8_t* gy, int hw, float* out, bool accumulate) -> int {
    return for_each_dgrad_launch(cw, 0, m.packed, gy, B, hw, hw, out, accumulate, [&](const dmd_conv_desc& d) { return dmd_conv2d_fprop(&d, st); });
  };
  // spatial size of every level's input
  std::vector<int> size_in(h->levels.size() + 1);
  { int S = c.img_size; for (size_t i = 0; i < h->levels.size(); ++i) { size_in[i] = S; if (h->levels[i].down) S /= 2; } size_in[h->levels.size()] = S; }
  for (int i = (int)h->levels.size() - 1; i >= 0; --i) {
    const auto& lv = h->levels[i];
    const int S = size_in[i];
    const float* gy = g_cur;            // gradient of the SmallResBlock output y[i] (NHWC, S x S x cout)
    float* gx = other(g_cur);           // gradient of the block input pooled[i]
    if (lv.down) {                      // un-pool into the other buffer; the pooled gradient's buffer then takes gx
      if (maxpool2_bwd_launch(b.y[i], g_cur, other(g_cur), B, S, S, lv.cout, st)) return 1;
      gy = other(g_cur);
      gx = g_cur;
    }
    const long long pix = (long long)B * S * S;
    // SmallResBlock (blocks.py:116-123): y = skip(x) + conv3x3(silu(GroupNorm(x)))
    dmd_prep_desc pd = prep_desc(gy, lv.cout, B, S, S, 0, 0, nullptr, nullptr, nullptr, sc.gy_op);
    if (dmd_prep_act(&pd, st)) return 1;
    if (colsum(gy, pix, lv.cout, lv.cout, G(lv.conv.b_idx), lv.has_skip ? G(lv.skip.b_idx) : nullptr, inv)) return 1;
    pd = prep_desc(b.pooled[i], lv.cin, B, S, S, 0, 2, b.st_in[i], m.P(lv.gn_w), m.P(lv.gn_b), sc.x_op);
    if (dmd_prep_act(&pd, st)) return 1;
    if (wgrad(lv.conv, sc.gy_op, sc.x_op, round_up(lv.cin, 16), S)) return 1;
    if (dgrad(lv.conv, sc.gy_op, S, sc.tA, false)) return 1;
    const NormBwdParams nb = gn_bwd_params(b.pooled[i], sc.tA, b.st_in[i], B, S * S, lv.cin, gn_group_size(lv.cin), m.P(lv.gn_w),
                                           m.P(lv.gn_b), sc.nsum, gx, lv.has_skip ? nullptr : gy, false);
    DMD_CUDA(cudaMemsetAsync(sc.nsum, 0, (size_t)2 * B * kMaxCin * 4, st));
    if (norm_bwd_launch(nb, 1, st, m.det) || affine_param_grad_launch(nb, G(lv.gn_w), G(lv.gn_b), inv, st) || norm_bwd_launch(nb, 2, st)) return 1;
    if (lv.has_skip) {  // 1x1 skip projection on the raw input
      pd = prep_desc(b.pooled[i], lv.cin, B, S, S, 0, 0, nullptr, nullptr, nullptr, sc.x_op);
      if (dmd_prep_act(&pd, st)) return 1;
      if (wgrad(lv.skip, sc.gy_op, sc.x_op, round_up(lv.cin, 16), S)) return 1;
      if (dgrad(lv.skip, sc.gy_op, S, gx, true)) return 1;
    }
    g_cur = gx;
  }
  {  // conv0 (Conv3x3(img_channels -> channels[0])): weight / bias gradients only
    const int S = c.img_size;
    dmd_prep_desc pd = prep_desc(g_cur, h->conv0.Cout, B, S, S, 0, 0, nullptr, nullptr, nullptr, sc.gy_op);
    if (dmd_prep_act(&pd, st)) return 1;
    if (colsum(g_cur, (long long)B * S * S, h->conv0.Cout, h->conv0.Cout, G(h->conv0.b_idx), nullptr, inv)) return 1;
    pd = prep_desc(b.x0, h->conv0.c0_store, B, S, S, 0, 0, nullptr, nullptr, nullptr, sc.x_op);
    if (dmd_prep_act(&pd, st)) return 1;
    if (wgrad(h->conv0, sc.gy_op, sc.x_op, h->conv0.c0_store, S)) return 1;
  }
  return 0;
}


// compute_lambda_returns (actor_critic.py:116-143) on the device, bit-identical to the torch expression (SURVEY.md 8 f4).
extern "C" int dmd_lambda_returns(const float* rew, const int64_t* end, const int64_t* trunc, const float* val_bootstrap, float* out,
                                  int B, int T, double gamma, double lambda_, void* stream) {
  DMD_CHECK(rew && end && trunc && val_bootstrap && out && B > 0 && T > 0, "lambda_returns: bad arguments");
  lambda_returns_kernel<<<(B + 127) / 128, 128, 0, (cudaStream_t)stream>>>(rew, (const long long*)end, (const long long*)trunc, val_bootstrap, out, B, T,
                                                                         (float)gamma, (float)lambda_, (float)(1.0 - lambda_));
  DMD_LAUNCH_OK();
  return 0;
}


// ---------------------------------------------------------------------------------------------- reward / termination model
// RewEndModel.predict_rew_end (src/models/rew_end_model.py:42-55; SURVEY.md 8 f1): runs once per imagined step between the
// sampler and the policy (world_model_env.py:97), and over the burn-in frames of every fresh episode (:120-129).
//   encoder (conv_in + ResBlocks at C = 32 conditioned on the action embedding + two attention ResBlocks) -> (b t) features
//   -> single-layer LSTM over time -> Linear / SiLU / Linear head -> 3 reward logits + 2 termination logits.
// Rows are processed TIME-MAJOR (row = k * b + n) so that every LSTM step reads b contiguous feature rows.  The handle
// (struct dmd_rew_end, next to dmd_denoiser) keeps the encoder plan of the last (rows, workspace) it ran.
namespace {

// obs / next_obs: (b, t, C, HW) fp32 (Obs = const float*), or frames (n, k) of two U8Frames sources (Obs = U8Frames)
template <class Obs>
__global__ void pack_rew_end_input_kernel(const Obs obs, const Obs next_obs, const int64_t* __restrict__ act,
                                          const float* __restrict__ act_emb, float* __restrict__ xin, float* __restrict__ cond,
                                          int64_t* __restrict__ act_tm, int b, int t, int C, int CP, int HW, int CC, int num_actions) {
  // row r = k * b + n (time-major)  <-  obs[n][k], next_obs[n][k], act[n][k]; act_tm (optional) [r] <- act[n][k]
  constexpr bool kU8 = std::is_same<Obs, U8Frames>::value;
  [[maybe_unused]] const float* tab = nullptr;
  if constexpr (kU8) tab = stage_decode_table(obs.table);   // both sources share one decode table (checked by the caller)
  const int r = blockIdx.y, k = r / b, n = r - k * b;
  const size_t src = ((size_t)n * t + k) * C * HW;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.x == 0) {
    long long a = act[(size_t)n * t + k];
    if (act_tm && threadIdx.x == 0) act_tm[r] = a;
    a = a < 0 ? 0 : (a >= num_actions ? num_actions - 1 : a);
    for (int j = threadIdx.x; j < CC; j += blockDim.x) cond[(size_t)r * CC + j] = act_emb[(size_t)a * CC + j];
  }
  if (pix >= HW) return;
  float* o = xin + ((size_t)r * HW + pix) * CP;
  for (int ch = 0; ch < CP; ++ch) {
    float v = 0.f;
    if constexpr (kU8) {
      if (ch < C) v = u8_frame_value(obs, tab, n, k, (size_t)ch * HW + pix);
      else if (ch < 2 * C) v = u8_frame_value(next_obs, tab, n, k, (size_t)(ch - C) * HW + pix);
    } else {
      if (ch < C) v = obs[src + (size_t)ch * HW + pix];
      else if (ch < 2 * C) v = next_obs[src + (size_t)(ch - C) * HW + pix];
    }
    o[ch] = v;
  }
}
// logits_tm [t*b][5] (time-major) -> rew [b][t][3], end [b][t][2]
__global__ void split_logits_kernel(const float* __restrict__ tm, float* __restrict__ rew, float* __restrict__ end, int b, int t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b * t) return;
  const int n = i / t, k = i - n * t;
  const float* s = tm + ((size_t)k * b + n) * 5;
  rew[(size_t)i * 3] = s[0]; rew[(size_t)i * 3 + 1] = s[1]; rew[(size_t)i * 3 + 2] = s[2];
  end[(size_t)i * 2] = s[3]; end[(size_t)i * 2 + 1] = s[4];
}
// the adjoint of split_logits_kernel: g_rew [b][t][3], g_end [b][t][2] -> time-major [t*b][5]
__global__ void merge_logits_kernel(const float* __restrict__ g_rew, const float* __restrict__ g_end, float* __restrict__ tm, int b, int t) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b * t) return;
  const int n = i / t, k = i - n * t;
  float* d = tm + ((size_t)k * b + n) * 5;
  d[0] = g_rew[(size_t)i * 3]; d[1] = g_rew[(size_t)i * 3 + 1]; d[2] = g_rew[(size_t)i * 3 + 2];
  d[3] = g_end[(size_t)i * 2]; d[4] = g_end[(size_t)i * 2 + 1];
}

// the encoder plan for B rows on the workspace at base (a first pass on null bases sizes the statistics region), then the LSTM /
// head buffers behind it.  base == nullptr: sizes only (*total)
int rew_end_layout(const dmd_rew_end* h, int B, uint8_t* base, RewEndLayout* o, size_t* total) {
  const int S = h->cfg.img_size;
  Plan& pl = o->plan;
  pl.train = false; pl.B = B; pl.H = S; pl.W = S; pl.det = h->core.det; pl.ops.clear();
  Bump b0{nullptr}, s0{nullptr};
  { Plan tmp; tmp.B = B; tmp.H = S; tmp.W = S; tmp.det = h->core.det; PlanBuilder pb{&h->core, &tmp, &b0, &s0}; if (pb.build_rew_end(h, &o->feat)) return 1; }
  const size_t stats_bytes = (s0.off + 255) & ~(size_t)255;
  Bump sb{base}, bb{base ? base + stats_bytes : nullptr};
  if (base) {
    pl.base = base; pl.stats = (double*)base; pl.stats_bytes = stats_bytes;
    PlanBuilder pb{&h->core, &pl, &bb, &sb};
    if (pb.build_rew_end(h, &o->feat)) return 1;
  } else bb.off = b0.off;
  const int D = h->cfg.lstm_dim;
  o->x_gates = (float*)bb.take((size_t)B * 4 * D * 4);
  o->y = (float*)bb.take((size_t)B * D * 4); o->hid = (float*)bb.take((size_t)B * D * 4);
  o->logits_tm = (float*)bb.take((size_t)B * 5 * 4);
  o->hc[0] = (float*)bb.take((size_t)B * D * 4); o->hc[1] = (float*)bb.take((size_t)B * D * 4);
  if (total) *total = stats_bytes + bb.off + 512;
  return 0;
}

// training workspace of b segments x t steps: the encoder plan with its gradients and backward temporaries
// (make_train_plan), plus the LSTM / head tape and the temporaries of their backward
int make_rew_end_train_plan(const dmd_rew_end* h, Plan* pl, int b, int t, uint8_t* base, size_t* total) {
  const int S = h->cfg.img_size, D = h->cfg.lstm_dim;
  auto fwd = [h, b, t, D](PlanBuilder& pb) {
    Plan* p = pb.pl;
    if (pb.build_rew_end(h, &p->feat)) return 1;
    const size_t rows = (size_t)b * t, state = (rows + b) * D * 4;
    Bump& m = *pb.bump;
    p->gates = (float*)m.take(rows * 4 * D * 4); p->cseq = (float*)m.take(state); p->hseq = (float*)m.take(state);
    p->hid = (float*)m.take(rows * D * 4); p->logits_tm = (float*)m.take(rows * 5 * 4); p->act_tm = (int64_t*)m.take(rows * 8);
    p->g_tm = (float*)m.take(rows * 5 * 4); p->g_hid = (float*)m.take(rows * D * 4); p->hpre = (float*)m.take(rows * D * 4);
    p->g_pre = (float*)m.take(rows * D * 4); p->g_y = (float*)m.take(rows * D * 4); p->dgates = (float*)m.take(rows * 4 * D * 4);
    p->gcs = (float*)m.take((size_t)2 * b * D * 4);
    return 0;
  };
  // the encoder's output gradient is seeded by the LSTM backward; the FiLM rows read act_emb(act) directly
  // (rew_end_model.py:51, no conditioning MLP), so the conditioning path ends in the embedding
  auto bwd = [h](BwdBuilder& bw) {
    bw.begin();
    bw.ginit[bw.pl->feat.gid] = 1;
    if (bw.walk((int)bw.pl->tape.size())) return 1;
    bw.film_tail();
    bw.embedding(bw.pl->dcond, h->i_actemb, 1, h->cfg.num_actions);
    return bw.err;
  };
  return make_train_plan(h->core, widest_channels(h->cfg), 0, pl, b * t, S, S, t, base, total, fwd, bwd);
}

// the encoder over the b * t time-major rows of pl: inputs, action embedding (act_tm, optional: a time-major copy of the
// actions), all FiLM rows, then the plan's ops.  u8 != null: u8[0] / u8[1] are the uint8 obs / next_obs (obs, next_obs unused)
int rew_end_encode(const dmd_rew_end* h, Plan& pl, int b, int t, const float* obs, const float* next_obs, const int64_t* act,
                   int64_t* act_tm, cudaStream_t st, const U8Frames* u8 = nullptr) {
  const ModelCore& m = h->core;
  const dmd_rew_end_config& c = h->cfg;
  const int rows = b * t, HW = c.img_size * c.img_size;
  DMD_CUDA(cudaMemsetAsync(pl.stats, 0, pl.stats_bytes, st));
  const dim3 grid((HW + 255) / 256, rows);
  if (u8)
    pack_rew_end_input_kernel<<<grid, 256, 0, st>>>(u8[0], u8[1], act, m.ptrs[h->i_actemb], pl.xin, pl.cond, act_tm,
                                                    b, t, c.img_channels, pl.CP_in, HW, c.cond_channels, c.num_actions);
  else
    pack_rew_end_input_kernel<<<grid, 256, 0, st>>>(obs, next_obs, act, m.ptrs[h->i_actemb], pl.xin, pl.cond, act_tm,
                                                    b, t, c.img_channels, pl.CP_in, HW, c.cond_channels, c.num_actions);
  DMD_LAUNCH_OK();
  if (linear_launch(pl.cond, (const float*)(m.packed + m.film_w_off), (const float*)(m.packed + m.film_b_off), pl.film,
                    rows, c.cond_channels, m.film_rows, 0, st)) return 1;
  for (const Op& op : pl.ops) {
    if (op.kind == OP_CONV) { if (conv_launch(op.conv, op.smem, op.cols, st)) return 1; }
    else if (op.kind == OP_PREP) { if (prep_launch(op.prep, op.prep_nsrc, st)) return 1; }
    else if (op.kind == OP_STATS) { if (gn_stats_launch(op.gn.x, op.gn.stats, pl.B, op.gn.HW, op.gn.C, op.gn.gs, pl.det, st)) return 1; }
    else { if (attn_launch(op.attn, pl.B, st)) return 1; }
  }
  return 0;
}

// LSTM over time (torch.nn.LSTM, gate order i f g o), rows of step k are the contiguous block [k*b, (k+1)*b).  gates: one
// [b][4D] buffer for every step, or (keep_gates) [t][b][4D]; y [t][b][D] receives h_1 ... h_t; c_seq [t][b][D] receives
// c_1 ... c_t, or (NULL) every step updates c_last in place
int rew_end_lstm(const dmd_rew_end* h, int b, int t, const float* feat, float* gates, bool keep_gates, const float* h0, const float* c0,
                 float* y, float* c_seq, float* c_last, cudaStream_t st) {
  const ModelCore& m = h->core;
  const int D = h->cfg.lstm_dim, K = h->feat_c * h->feat_hw;
  const float* hprev = h0; const float* cprev = c0;
  for (int k = 0; k < t; ++k) {
    const float* xk = feat + (size_t)k * b * K;
    float* gk = keep_gates ? gates + (size_t)k * b * 4 * D : gates;
    if (linear_launch(xk, m.ptrs[h->i_wih], m.ptrs[h->i_bih], gk, b, K, 4 * D, 0, st, 0, h->feat_hw)) return 1;
    if (linear_launch(hprev, m.ptrs[h->i_whh], m.ptrs[h->i_bhh], gk, b, D, 4 * D, 0, st, 1, 0)) return 1;
    float* hk = y + (size_t)k * b * D;   // y rows of step k (time-major); also the next step's h
    float* ck = c_seq ? c_seq + (size_t)k * b * D : c_last;
    if (lstm_gates_launch(gk, cprev, hk, ck, b, D, st)) return 1;
    hprev = hk; cprev = ck;
  }
  return 0;
}

// head: Linear(D, D) + SiLU + Linear(D, 5, bias=False) over all rows, then the split into (b, t, 3) and (b, t, 2)
int rew_end_head(const dmd_rew_end* h, int b, int t, const float* y, float* hid, float* logits_tm, float* logits_rew, float* logits_end,
                 cudaStream_t st) {
  const ModelCore& m = h->core;
  const int rows = b * t, D = h->cfg.lstm_dim;
  if (linear_launch(y, m.ptrs[h->i_h0w], m.ptrs[h->i_h0b], hid, rows, D, D, 1, st)) return 1;
  if (linear_launch(hid, m.ptrs[h->i_h2w], nullptr, logits_tm, rows, D, 5, 0, st)) return 1;
  split_logits_kernel<<<(rows + 127) / 128, 128, 0, st>>>(logits_tm, logits_rew, logits_end, b, t);
  DMD_LAUNCH_OK();
  return 0;
}

}  // namespace

extern "C" dmd_rew_end* dmd_rew_end_create(const dmd_rew_end_config* cfg) {
  if (!cfg || cfg->num_levels < 1 || cfg->num_levels >= DMD_MAX_LEVELS) { fail("rew_end_create: bad config"); return nullptr; }
  if (cfg->cond_channels <= 0 || cfg->cond_channels % 32 || cfg->cond_channels > kMaxCondChannels) {
    fail("rew_end_create: cond_channels must be a multiple of 32, at most %d; got %d", kMaxCondChannels, cfg->cond_channels);
    return nullptr;
  }
  for (int i = 0; i < cfg->num_levels; ++i)
    if (!level_width_ok(cfg->channels[i])) { fail("rew_end_create: channels must be 32, 64 or 128 per level, at most 128 (got %d at level %d)", cfg->channels[i], i); return nullptr; }
  if (cfg->lstm_dim % 4) { fail("rew_end_create: lstm_dim must be a multiple of 4"); return nullptr; }
  if (init_kernels()) return nullptr;
  dmd_rew_end* h = new dmd_rew_end();
  h->cfg = *cfg;
  h->core.cond_channels = cfg->cond_channels;
  // registration order (rew_end_model.py:27-41, :93-125): encoder.{conv_in, blocks[0..L], downsamples[1..L-1]}, act_emb, lstm, head
  Walker w{&h->core};
  const int L = cfg->num_levels;
  const int cin_real = 2 * cfg->img_channels;
  h->conv_in = w.conv(cfg->channels[0], cin_real, 9, cin_real, round_up(cin_real, 16), 0, true, false);
  h->blocks.resize(L + 1);
  for (int i = 0; i < L; ++i) {
    const int c1 = cfg->channels[i > 0 ? i - 1 : 0], c2 = cfg->channels[i];
    for (int k = 0; k < cfg->depths[i]; ++k) h->blocks[i].push_back(w.resblock(k == 0 ? c1 : c2, 0, c2, cfg->attn_depths[i] != 0));
  }
  for (int k = 0; k < 2; ++k) h->blocks[L].push_back(w.resblock(cfg->channels[L - 1], 0, cfg->channels[L - 1], true));
  h->downs.resize(L);
  for (int i = 1; i < L; ++i) h->downs[i] = w.conv(cfg->channels[i - 1], cfg->channels[i - 1], 9, cfg->channels[i - 1], cfg->channels[i - 1], 0);
  const int S = cfg->img_size >> (L - 1);
  h->feat_c = cfg->channels[L - 1]; h->feat_hw = S * S;
  const long long D = cfg->lstm_dim, K = (long long)h->feat_c * h->feat_hw;
  h->i_actemb = w.next((long long)cfg->num_actions * cfg->cond_channels);
  h->i_wih = w.next(4 * D * K); h->i_whh = w.next(4 * D * D); h->i_bih = w.next(4 * D); h->i_bhh = w.next(4 * D);
  h->i_h0w = w.next(D * D); h->i_h0b = w.next(D); h->i_h2w = w.next(5 * D);
  h->core.finish(w.pk);
  if (w.err) { delete h; return nullptr; }
  return h;
}
extern "C" void dmd_rew_end_destroy(dmd_rew_end* h) { delete h; }
extern "C" int dmd_rew_end_num_tensors(const dmd_rew_end* h) { return h->core.n_tensors; }
extern "C" size_t dmd_rew_end_packed_bytes(const dmd_rew_end* h) { return h->core.packed_bytes; }

static int pack_rew_end(const dmd_rew_end* h, cudaStream_t st) {
  const ModelCore& m = h->core;
  if (pack_one(m, h->conv_in, st)) return 1;
  for (auto& lv : h->blocks) for (auto& r : lv) if (pack_rb(m, r, st)) return 1;
  for (int i = 1; i < h->cfg.num_levels; ++i) if (pack_one(m, h->downs[i], st)) return 1;
  return 0;
}

extern "C" int dmd_rew_end_set_weights(dmd_rew_end* h, const float* const* ptrs_host, int n_ptrs, void* packed, void* stream) {
  DMD_CHECK(h, "set_weights: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  bool moved = false, pack_now = false;
  if (h->core.set_weights("RewEndModel", ptrs_host, n_ptrs, packed, &moved)) return 1;
  if (moved) { h->lay.plan.B = 0; h->core.tplans.clear(); }   // plans bake parameter and packed-weight addresses in
  if (set_weights_tail(h->core, st, &pack_now)) return 1;
  return pack_now ? pack_rew_end(h, st) : 0;
}

extern "C" size_t dmd_rew_end_workspace_bytes(const dmd_rew_end* h, int rows) {
  RewEndLayout tmp; size_t total = 0;
  if (rew_end_layout(h, rows, nullptr, &tmp, &total)) return 0;
  return total;
}

// obs / next_obs (b, t, C, S, S) fp32, act (b, t) int64, hx_in / cx_in (b, lstm_dim) or NULL (zeros).
// Outputs: logits_rew (b, t, 3), logits_end (b, t, 2), hx_out / cx_out (b, lstm_dim).
namespace {
int rew_end_predict(dmd_rew_end* h, int b, int t, const float* obs, const float* next_obs, const U8Frames* u8, const int64_t* act,
                    const float* hx_in, const float* cx_in, float* logits_rew, float* logits_end, float* hx_out,
                    float* cx_out, void* workspace, size_t workspace_bytes, void* stream) {
  const ModelCore& m = h->core;
  DMD_CHECK(m.ready(), "rew_end predict: call dmd_rew_end_set_weights first");
  DMD_CHECK(((uintptr_t)workspace & 255) == 0, "rew_end predict: workspace must be 256-byte aligned");
  const dmd_rew_end_config& c = h->cfg;
  cudaStream_t st = (cudaStream_t)stream;
  const int rows = b * t, D = c.lstm_dim;
  RewEndLayout& o = h->lay;
  Plan& pl = o.plan;
  if (pl.B != rows || pl.base != (uint8_t*)workspace || pl.det != h->core.det) {
    // size and validate on a scratch layout; the cached one is invalidated (never left half-written) if the real build fails
    size_t need = 0;
    { RewEndLayout tmp; if (rew_end_layout(h, rows, nullptr, &tmp, &need)) return 1; }
    DMD_CHECK(workspace_bytes >= need, "rew_end predict: workspace too small (%zu < %zu)", workspace_bytes, need);
    if (rew_end_layout(h, rows, (uint8_t*)workspace, &o, nullptr)) { pl.B = 0; pl.base = nullptr; pl.ops.clear(); return 1; }
  }
  bool cap = false;
  if (stream_capturing(st, &cap) || (cap && pack_rew_end(h, st))) return 1;
  if (rew_end_encode(h, pl, b, t, obs, next_obs, act, nullptr, st, u8)) return 1;
  const float* hprev = hx_in; const float* cprev = cx_in;
  if (!hx_in) { DMD_CUDA(cudaMemsetAsync(o.hc[0], 0, (size_t)b * D * 4, st)); hprev = o.hc[0]; }
  if (!cx_in) { DMD_CUDA(cudaMemsetAsync(o.hc[1], 0, (size_t)b * D * 4, st)); cprev = o.hc[1]; }
  if (rew_end_lstm(h, b, t, o.feat.data, o.x_gates, false, hprev, cprev, o.y, nullptr, cx_out, st)) return 1;
  DMD_CUDA(cudaMemcpyAsync(hx_out, o.y + (size_t)(t - 1) * b * D, (size_t)b * D * 4, cudaMemcpyDeviceToDevice, st));
  return rew_end_head(h, b, t, o.y, o.hid, o.logits_tm, logits_rew, logits_end, st);
}

// the pointer arguments every reward / termination entry point shares, each named in its message
int rew_end_args(const char* who, const dmd_rew_end* h, int b, int t, const int64_t* act, const float* logits_rew, const float* logits_end,
                 const float* hx_out, const float* cx_out, const void* workspace) {
  DMD_CHECK(h, "%s: handle is NULL", who);
  DMD_CHECK(b > 0 && t > 0, "%s: bad shape b=%d t=%d", who, b, t);
  DMD_CHECK(act, "%s: act is NULL", who);
  DMD_CHECK(logits_rew && logits_end, "%s: logits_rew / logits_end is NULL", who);
  DMD_CHECK(hx_out && cx_out, "%s: hx_out / cx_out is NULL", who);
  DMD_CHECK(workspace, "%s: workspace is NULL", who);
  return 0;
}

// both uint8 sources of a reward / termination call; they share one decode table
int rew_end_u8_args(const char* who, const dmd_u8_frames* obs, const dmd_u8_frames* next_obs, U8Frames* out) {
  if (u8_frames_arg(who, "obs", obs, &out[0]) || u8_frames_arg(who, "next_obs", next_obs, &out[1])) return 1;
  DMD_CHECK(obs->table == next_obs->table, "%s: obs->table and next_obs->table differ (the sources share one decode table)", who);
  return 0;
}
}  // namespace

extern "C" int dmd_rew_end_predict(dmd_rew_end* h, int b, int t, const float* obs, const float* next_obs, const int64_t* act,
                                   const float* hx_in, const float* cx_in, float* logits_rew, float* logits_end, float* hx_out,
                                   float* cx_out, void* workspace, size_t workspace_bytes, void* stream) {
  DMD_CHECK(h && obs && next_obs && act && logits_rew && logits_end && hx_out && cx_out && workspace, "rew_end predict: null argument");
  return rew_end_predict(h, b, t, obs, next_obs, nullptr, act, hx_in, cx_in, logits_rew, logits_end, hx_out, cx_out, workspace,
                         workspace_bytes, stream);
}

extern "C" int dmd_rew_end_predict_u8(dmd_rew_end* h, int b, int t, const dmd_u8_frames* obs, const dmd_u8_frames* next_obs,
                                      const int64_t* act, const float* hx_in, const float* cx_in, float* logits_rew, float* logits_end,
                                      float* hx_out, float* cx_out, void* workspace, size_t workspace_bytes, void* stream) {
  const char* who = "rew_end_predict_u8";
  if (rew_end_args(who, h, b, t, act, logits_rew, logits_end, hx_out, cx_out, workspace)) return 1;
  U8Frames u8[2];
  if (rew_end_u8_args(who, obs, next_obs, u8)) return 1;
  return rew_end_predict(h, b, t, nullptr, nullptr, u8, act, hx_in, cx_in, logits_rew, logits_end, hx_out, cx_out, workspace,
                         workspace_bytes, stream);
}

// ---------------------------------------------------------------------------------------------- reward / termination training
// RewEndModel.forward (rew_end_model.py:57-90) under autograd: dmd_rew_end_forward_train is dmd_rew_end_predict that keeps the
// encoder's activations, every LSTM step's gates and states and the head's hidden layer in a training workspace;
// dmd_rew_end_backward runs the head and the LSTM (BPTT) backward, then the encoder's backward op list (BwdBuilder, shared
// with the denoiser) and the FiLM / action-embedding tail.
extern "C" size_t dmd_rew_end_train_workspace_bytes(const dmd_rew_end* h, int b, int t) {
  if (!h || b <= 0 || t <= 0) { fail("rew_end_train_workspace_bytes: bad arguments"); return 0; }
  Plan tmp; size_t need = 0;
  if (make_rew_end_train_plan(h, &tmp, b, t, nullptr, &need)) return 0;
  return need;
}
extern "C" long long dmd_rew_end_grad_layout(const dmd_rew_end* h, long long* offsets, long long* numels, int n) {
  return grad_layout(h ? &h->core : nullptr, offsets, numels, n);
}

namespace {
int rew_end_forward_train(dmd_rew_end* h, int b, int t, const float* obs, const float* next_obs, const U8Frames* u8, const int64_t* act,
                          const float* hx_in, const float* cx_in, float* logits_rew, float* logits_end, float* hx_out,
                          float* cx_out, void* workspace, size_t workspace_bytes, void* stream) {
  const int S = h->cfg.img_size, D = h->cfg.lstm_dim;
  cudaStream_t st = (cudaStream_t)stream;
  Plan* pl = nullptr;
  auto make = [h, b, t](Plan* p, uint8_t* base, size_t* total) { return make_rew_end_train_plan(h, p, b, t, base, total); };
  if (ensure_train_plan(h->core, "rew_end", b * t, S, S, t, workspace, workspace_bytes, make, &pl)) return 1;
  pl->t_act = pl->act_tm;
  if (rew_end_encode(h, *pl, b, t, obs, next_obs, act, pl->act_tm, st, u8)) return 1;
  // hseq = [h_in; y], cseq = [c_in; c_1 ... c_t]
  const size_t state = (size_t)b * D * 4;
  if (hx_in) DMD_CUDA(cudaMemcpyAsync(pl->hseq, hx_in, state, cudaMemcpyDeviceToDevice, st)); else DMD_CUDA(cudaMemsetAsync(pl->hseq, 0, state, st));
  if (cx_in) DMD_CUDA(cudaMemcpyAsync(pl->cseq, cx_in, state, cudaMemcpyDeviceToDevice, st)); else DMD_CUDA(cudaMemsetAsync(pl->cseq, 0, state, st));
  float* y = pl->hseq + (size_t)b * D;
  if (rew_end_lstm(h, b, t, pl->feat.data, pl->gates, true, pl->hseq, pl->cseq, y, pl->cseq + (size_t)b * D, nullptr, st)) return 1;
  DMD_CUDA(cudaMemcpyAsync(hx_out, pl->hseq + (size_t)t * b * D, state, cudaMemcpyDeviceToDevice, st));
  DMD_CUDA(cudaMemcpyAsync(cx_out, pl->cseq + (size_t)t * b * D, state, cudaMemcpyDeviceToDevice, st));
  return rew_end_head(h, b, t, y, pl->hid, pl->logits_tm, logits_rew, logits_end, st);
}
}  // namespace

extern "C" int dmd_rew_end_forward_train(dmd_rew_end* h, int b, int t, const float* obs, const float* next_obs, const int64_t* act,
                                         const float* hx_in, const float* cx_in, float* logits_rew, float* logits_end, float* hx_out,
                                         float* cx_out, void* workspace, size_t workspace_bytes, void* stream) {
  DMD_CHECK(h && obs && next_obs && act && logits_rew && logits_end && hx_out && cx_out && workspace, "rew_end forward_train: null argument");
  DMD_CHECK(b > 0 && t > 0, "rew_end forward_train: bad shape b=%d t=%d", b, t);
  return rew_end_forward_train(h, b, t, obs, next_obs, nullptr, act, hx_in, cx_in, logits_rew, logits_end, hx_out, cx_out, workspace,
                               workspace_bytes, stream);
}

extern "C" int dmd_rew_end_forward_train_u8(dmd_rew_end* h, int b, int t, const dmd_u8_frames* obs, const dmd_u8_frames* next_obs,
                                            const int64_t* act, const float* hx_in, const float* cx_in, float* logits_rew,
                                            float* logits_end, float* hx_out, float* cx_out, void* workspace, size_t workspace_bytes,
                                            void* stream) {
  const char* who = "rew_end_forward_train_u8";
  if (rew_end_args(who, h, b, t, act, logits_rew, logits_end, hx_out, cx_out, workspace)) return 1;
  U8Frames u8[2];
  if (rew_end_u8_args(who, obs, next_obs, u8)) return 1;
  return rew_end_forward_train(h, b, t, nullptr, nullptr, u8, act, hx_in, cx_in, logits_rew, logits_end, hx_out, cx_out, workspace,
                               workspace_bytes, stream);
}

namespace {
int rew_end_backward_impl(const char* who, dmd_rew_end* h, int b, int t, const float* g_logits_rew, const float* g_logits_end,
                          const float* g_hx_out, const float* g_cx_out, float* grads, long long grads_numel, int accumulate,
                          float* g_hx_in, float* g_cx_in, void* workspace, void* stream) {
  DMD_CHECK(h && g_logits_rew && g_logits_end && grads && workspace, "%s: null argument", who);
  const dmd_rew_end_config& c = h->cfg;
  Plan* plp = (b > 0 && t > 0) ? find_train_plan(h->core, b * t, c.img_size, c.img_size, t, workspace, true) : nullptr;
  DMD_CHECK(plp && plp->train, "%s: no matching dmd_rew_end_forward_train on this workspace (b=%d t=%d)", who, b, t);
  const ModelCore& m = h->core;
  DMD_CHECK(grads_numel >= m.grad_total, "%s: gradient buffer too small (%lld < %lld floats)", who, grads_numel, m.grad_total);
  DMD_CHECK(((uintptr_t)grads & 15) == 0, "%s: gradient buffer must be 16-byte aligned", who);
  Plan& pl = *plp;
  cudaStream_t st = (cudaStream_t)stream;
  const int rows = b * t, D = c.lstm_dim, K = h->feat_c * h->feat_hw;
  auto G = [&](int idx) { return grads + m.goff[idx]; };
  auto sgemm = [&](const float* Am, long long sam, long long sak, const float* Bm, long long sbk, long long sbn, float* C, long long ldc,
                   int M, int N, int Kd, int acc) -> int {
    return sgemm_launch(Am, sam, sak, Bm, sbk, sbn, C, ldc, M, N, Kd, nullptr, acc, 0, nullptr, st);
  };
  // every write into `grads` below adds to it (sgemm with acc = 1, colsum), as run_backward's do
  if (clear_backward(m, pl, grads, accumulate, st)) return 1;
  // ---- head (rew_end_model.py:54): logits = W2 silu(W0 y + b0); these gradients are fp32 and unscaled
  const float* y = pl.hseq + (size_t)b * D;
  merge_logits_kernel<<<(rows + 127) / 128, 128, 0, st>>>(g_logits_rew, g_logits_end, pl.g_tm, b, t);
  DMD_LAUNCH_OK();
  if (sgemm(pl.g_tm, 1, 5, pl.hid, D, 1, G(h->i_h2w), D, 5, D, rows, 1)) return 1;                // dW2 += g^T hid
  if (sgemm(pl.g_tm, 5, 1, m.ptrs[h->i_h2w], D, 1, pl.g_hid, D, rows, D, 5, 0)) return 1;          // g_hid = g W2
  if (linear_launch(y, m.ptrs[h->i_h0w], m.ptrs[h->i_h0b], pl.hpre, rows, D, D, 0, st)) return 1;  // the forward's pre-activation
  if (dsilu_mul_launch(pl.hpre, pl.g_hid, pl.g_pre, (long long)rows * D, st)) return 1;
  if (sgemm(pl.g_pre, 1, D, y, D, 1, G(h->i_h0w), D, D, D, rows, 1)) return 1;                    // dW0 += g_pre^T y
  if (colsum_launch(pl.g_pre, G(h->i_h0b), nullptr, nullptr, rows, D, D, st, pl.det ? pl.partial : nullptr, pl.partial_bytes)) return 1;
  if (sgemm(pl.g_pre, D, 1, m.ptrs[h->i_h0w], D, 1, pl.g_y, D, rows, D, D, 0)) return 1;          // g_y = g_pre W0
  // ---- LSTM (rew_end_model.py:53), back through time: g_h of step k = g_y[k] (+ g_hx_out at the last step) + dgates_{k+1} W_hh
  const float* Whh = m.ptrs[h->i_whh];
  if (g_hx_out) {   // g_y[t-1] += g_hx_out (a one-way split-K reduce)
    const long long n = (long long)b * D;
    splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g_hx_out, 1, n, pl.g_y + (size_t)(t - 1) * b * D, nullptr, 1);
    DMD_LAUNCH_OK();
  }
  for (int k = t - 1; k >= 0; --k) {
    const size_t r0 = (size_t)k * b;
    const float* g_c = k == t - 1 ? g_cx_out : pl.gcs + (size_t)((k + 1) & 1) * b * D;
    float* g_c_in = (k == 0 && g_cx_in) ? g_cx_in : pl.gcs + (size_t)(k & 1) * b * D;
    float* dg = pl.dgates + r0 * 4 * D;
    if (lstm_cell_bwd_launch(pl.gates + r0 * 4 * D, pl.cseq + r0 * D, pl.g_y + r0 * D, g_c, dg, g_c_in, b, D, st)) return 1;
    if (k > 0) { if (sgemm(dg, 4 * D, 1, Whh, D, 1, pl.g_y + (r0 - b) * D, D, b, D, 4 * D, 1)) return 1; }   // g_y[k-1] += dgates_k W_hh
    else if (g_hx_in && sgemm(dg, 4 * D, 1, Whh, D, 1, g_hx_in, D, b, D, 4 * D, 0)) return 1;                  // g_hx_in = dgates_0 W_hh
  }
  // input / recurrent weights over all t*b rows at once; x: the NCHW flatten of the features (rew_end_model.py:52)
  float* x_flat = pl.tB;
  float* g_x = pl.tC;
  if (dmd_nhwc_to_nchw(pl.feat.data, x_flat, rows, h->feat_c, h->feat_c, h->feat_hw, st)) return 1;
  if (sgemm(pl.dgates, 1, 4 * D, x_flat, K, 1, G(h->i_wih), K, 4 * D, K, rows, 1)) return 1;     // dW_ih += dgates^T x
  if (sgemm(pl.dgates, 1, 4 * D, pl.hseq, D, 1, G(h->i_whh), D, 4 * D, D, rows, 1)) return 1;    // dW_hh += dgates^T [h_in; y[:-1]]
  if (colsum_launch(pl.dgates, G(h->i_bih), G(h->i_bhh), nullptr, rows, 4 * D, 4 * D, st, pl.det ? pl.partial : nullptr, pl.partial_bytes)) return 1;
  if (sgemm(pl.dgates, 4 * D, 1, m.ptrs[h->i_wih], K, 1, g_x, K, rows, K, 4 * D, 0)) return 1;   // g_x = dgates W_ih
  // ---- encoder: the feature gradient enters the fp16 tensor-core path with a loss scale, NHWC in the last tensor's gradient
  if (loss_scale_launch(g_x, (long long)rows * K, pl.amax, pl.scale, st)) return 1;
  nchw_to_nhwc_scaled_kernel<<<dim3((h->feat_hw + 255) / 256, rows), 256, 0, st>>>(g_x, pl.feat.grad, pl.scale, h->feat_c, h->feat_c, h->feat_hw);
  DMD_LAUNCH_OK();
  return run_backward(m, pl, grads, st);
}
}  // namespace

extern "C" int dmd_rew_end_backward(dmd_rew_end* h, int b, int t, const float* g_logits_rew, const float* g_logits_end,
                                    const float* g_hx_out, const float* g_cx_out, float* grads, long long grads_numel,
                                    float* g_hx_in, float* g_cx_in, void* workspace, void* stream) {
  return rew_end_backward_impl("rew_end backward", h, b, t, g_logits_rew, g_logits_end, g_hx_out, g_cx_out, grads, grads_numel, 0,
                               g_hx_in, g_cx_in, workspace, stream);
}
extern "C" int dmd_rew_end_backward_accumulate(dmd_rew_end* h, int b, int t, const float* g_logits_rew, const float* g_logits_end,
                                               const float* g_hx_out, const float* g_cx_out, float* grads, long long grads_numel,
                                               float* g_hx_in, float* g_cx_in, void* workspace, void* stream) {
  return rew_end_backward_impl("rew_end backward_accumulate", h, b, t, g_logits_rew, g_logits_end, g_hx_out, g_cx_out, grads,
                               grads_numel, 1, g_hx_in, g_cx_in, workspace, stream);
}

// ---------------------------------------------------------------------------------------------- optimizer (optim_kernels.cuh)
// clip_grad_norm_ + AdamW over a caller's tensor table (dmd_optim_tensor, host memory): the table is checked whole before any
// CUDA call, then cut into launches of at most kOptMaxTensors non-empty tensors.

static int optim_check_table(const dmd_optim_tensor* t, int n, bool adamw, const char* who) {
  DMD_CHECK(t, "%s: null tensor table", who);
  DMD_CHECK(((uintptr_t)t % alignof(dmd_optim_tensor)) == 0, "%s: misaligned tensor table (needs %d-byte alignment)", who,
            (int)alignof(dmd_optim_tensor));
  DMD_CHECK(n > 0, "%s: n = %d tensors (need n > 0)", who, n);
  for (int i = 0; i < n; ++i) {
    const dmd_optim_tensor& e = t[i];
    DMD_CHECK(e.numel >= 0, "%s: tensor %d has negative numel %lld", who, i, e.numel);
    DMD_CHECK(e.numel < (1ll << 40), "%s: tensor %d numel %lld too large", who, i, e.numel);
    if (e.numel == 0) continue;
    DMD_CHECK(e.grad, "%s: tensor %d has a null grad pointer", who, i);
    DMD_CHECK(((uintptr_t)e.grad & 3) == 0, "%s: tensor %d grad pointer not 4-byte aligned", who, i);
    if (!adamw) continue;
    DMD_CHECK(e.param && e.exp_avg && e.exp_avg_sq, "%s: tensor %d has a null param / exp_avg / exp_avg_sq pointer", who, i);
    DMD_CHECK((((uintptr_t)e.param | (uintptr_t)e.exp_avg | (uintptr_t)e.exp_avg_sq) & 3) == 0,
              "%s: tensor %d param / exp_avg / exp_avg_sq pointer not 4-byte aligned", who, i);
    DMD_CHECK(std::isfinite(e.weight_decay) && e.weight_decay >= 0, "%s: tensor %d weight_decay %g is not finite and >= 0", who, i,
              e.weight_decay);
  }
  return 0;
}

// Splits the table into launches; for each, fills `tab` and calls launch(tab, blocks, first_block).  Returns total blocks.
template <class F>
static long long optim_for_each_launch(const dmd_optim_tensor* t, int n, bool adamw, double lr, OptTable& tab, F&& launch) {
  long long total = 0;
  int i = 0;
  while (i < n) {
    tab.count = 0;
    int blocks = 0;
    for (; i < n && tab.count < kOptMaxTensors; ++i) {
      const dmd_optim_tensor& e = t[i];
      if (e.numel == 0) continue;
      const int k = tab.count++;
      tab.p[k] = e.param; tab.g[k] = e.grad; tab.m[k] = e.exp_avg; tab.v[k] = e.exp_avg_sq;
      tab.n[k] = e.numel;
      tab.decay[k] = (adamw && e.weight_decay != 0) ? (float)(1.0 - lr * e.weight_decay) : 1.0f;
      uintptr_t bits = (uintptr_t)e.grad;
      if (adamw) bits |= (uintptr_t)e.param | (uintptr_t)e.exp_avg | (uintptr_t)e.exp_avg_sq;
      tab.vec[k] = (bits & 15) == 0;
      tab.block0[k] = blocks;
      blocks += (int)((e.numel + kOptChunk - 1) / kOptChunk);
    }
    if (tab.count == 0) break;
    if (launch(tab, blocks, total)) return -1;
    total += blocks;
  }
  return total;
}

static long long optim_norm_blocks(const dmd_optim_tensor* t, int n) {
  static thread_local OptTable tab;
  return optim_for_each_launch(t, n, false, 0.0, tab, [](const OptTable&, int, long long) { return 0; });
}

extern "C" size_t dmd_grad_norm_partial_bytes(const dmd_optim_tensor* table_host, int n) {
  if (optim_check_table(table_host, n, false, "dmd_grad_norm_partial_bytes")) return 0;
  return (size_t)std::max(optim_norm_blocks(table_host, n), 1ll) * sizeof(double);
}

extern "C" int dmd_grad_norm_clip(const dmd_optim_tensor* table_host, int n, double max_norm, int clip, float* norm_coef,
                                  void* partial, size_t partial_bytes, void* stream) {
  if (optim_check_table(table_host, n, false, "dmd_grad_norm_clip")) return 1;
  DMD_CHECK(!std::isnan(max_norm) && max_norm >= 0, "dmd_grad_norm_clip: max_norm %g is not >= 0", max_norm);
  DMD_CHECK(norm_coef, "dmd_grad_norm_clip: null norm_coef");
  DMD_CHECK(partial, "dmd_grad_norm_clip: null partial buffer");
  DMD_CHECK(((uintptr_t)partial & 7) == 0, "dmd_grad_norm_clip: partial buffer not 8-byte aligned");
  const long long blocks = optim_norm_blocks(table_host, n);
  DMD_CHECK(partial_bytes >= (size_t)std::max(blocks, 1ll) * sizeof(double),
            "dmd_grad_norm_clip: partial buffer too small (%zu < %zu bytes; dmd_grad_norm_partial_bytes)", partial_bytes,
            (size_t)std::max(blocks, 1ll) * sizeof(double));
  cudaStream_t st = (cudaStream_t)stream;
  double* part = (double*)partial;
  static thread_local OptTable tab;
  auto norm = [&](const OptTable& tb, int nb, long long first) -> int {
    grad_sqnorm_kernel<<<nb, kOptThreads, 0, st>>>(tb, part, (int)first);
    DMD_LAUNCH_OK();
    return 0;
  };
  if (optim_for_each_launch(table_host, n, false, 0.0, tab, norm) < 0) return 1;
  grad_norm_finalize_kernel<<<1, kOptThreads, 0, st>>>(part, (int)blocks, (float)max_norm, norm_coef);
  DMD_LAUNCH_OK();
  if (!clip) return 0;
  auto scale = [&](const OptTable& tb, int nb, long long) -> int {
    grad_scale_kernel<<<nb, kOptThreads, 0, st>>>(tb, norm_coef + 1);
    DMD_LAUNCH_OK();
    return 0;
  };
  return optim_for_each_launch(table_host, n, false, 0.0, tab, scale) < 0 ? 1 : 0;
}

extern "C" int dmd_adamw_step(const dmd_optim_tensor* table_host, int n, double lr, double beta1, double beta2, double eps,
                              double step, void* stream) {
  if (optim_check_table(table_host, n, true, "dmd_adamw_step")) return 1;
  DMD_CHECK(std::isfinite(lr) && lr >= 0, "dmd_adamw_step: lr %g is not finite and >= 0", lr);
  DMD_CHECK(std::isfinite(eps) && eps >= 0, "dmd_adamw_step: eps %g is not finite and >= 0", eps);
  DMD_CHECK(beta1 >= 0 && beta1 < 1 && beta2 >= 0 && beta2 < 1, "dmd_adamw_step: betas (%g, %g) not in [0, 1)", beta1, beta2);
  DMD_CHECK(std::isfinite(step) && step >= 1, "dmd_adamw_step: step %g is not finite and >= 1", step);
  // torch's Python-float arithmetic (adam.py, non-capturable branch), in double, then the fp32 values its kernels receive
  const double bc1 = 1.0 - std::pow(beta1, step), bc2 = 1.0 - std::pow(beta2, step);
  AdamWScalars s;
  s.w1 = (float)(1.0 - beta1);
  s.beta2 = (float)beta2;
  s.omb2 = (float)(1.0 - beta2);
  s.inv_bc2s = 1.0f / (float)std::pow(bc2, 0.5);
  s.eps = (float)eps;
  s.neg_step = (float)(-(lr / bc1));
  cudaStream_t st = (cudaStream_t)stream;
  static thread_local OptTable tab;
  auto launch = [&](const OptTable& tb, int nb, long long) -> int {
    adamw_kernel<<<nb, kOptThreads, 0, st>>>(tb, s);
    DMD_LAUNCH_OK();
    return 0;
  };
  return optim_for_each_launch(table_host, n, true, lr, tab, launch) < 0 ? 1 : 0;
}
