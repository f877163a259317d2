// Implicit-GEMM convolution on Hopper tensor cores (sm_90a wgmma).  Persistent, warp-specialised, TMA-fed.
//
// Replaces, on the hot path, every nn.Conv2d of the reference (blocks.py:18-19 Conv1x1/Conv3x3, :96 Downsample,
// :109-110 Upsample conv, inner_model.py:36,41 conv_in/conv_out) plus its epilogue neighbours: bias, residual add
// (blocks.py:145), stride-2 subsample (blocks.py:96) and the (sum, sumsq) partials of the NEXT GroupNorm.
// What the reference applies to the conv INPUT (GroupNorm / AdaGroupNorm + SiLU, concat, nearest-2x upsample) is done once
// per element by prep_act_kernel (below), which writes the activation operand in the layout this kernel consumes.
//
// Operand layout "PLC16" (padded-linear, chunk-major, fp16).  Pixels of all B images lie on one line with pitch
// PW = W+1 and PH = H+1 rows per image: q = (n*PH + y)*PW + x.  Column x==W and row y==H are zero padding shared
// between neighbouring rows / images, so tap (dy,dx) of a 3x3 window is simply position q + dy*PW + dx.  The tensor is
// stored as one plane per 8-channel chunk:   plane[j][G + q] = 8 fp16 channels = 16 bytes   (G = PW+1 zero guard
// positions in front, PW+1 behind the last tile).  A 128-row tile needs, per 16 input channels ("slab"), positions
// [q0-PW-1, q0+128+PW+1) of two planes: two CONTIGUOUS byte ranges.  They are fetched with cp.async.bulk straight
// into the wgmma no-swizzle K-major shared-memory layout  [2 chunks][P positions][16 B]  (LBO = Palloc*16, SBO = 128),
// and every tap reads the same slab through a descriptor whose start address is shifted by (dy*PW+dx)*16 B.
//
// Roles (384 threads = three warpgroups, one CTA per SM, contiguous balanced tile ranges):
//   warps 0, 1       producers: mbarrier expect_tx + 2 bulk copies per slab into a deep ring (empty/full mbarriers); the two
//                    warps take alternate slabs (warps 2 and 3 have no work)
//   warpgroups 1, 2  consumers: warpgroup c owns rows 64c .. 64c+63 of the tile.  Per (slab, tap) one wgmma m64 x N x k16 with
//                    both operands in shared memory and the fp32 accumulator in registers; a fused 1x1 skip projection is
//                    extra centre-tap slabs on the same accumulator.  After the last slab of a tile the warpgroup stores its
//                    rows (+bias, +residual) from the registers straight to NHWC global memory (RegEpilogue) while the
//                    producers already fill the ring with the next tile's slabs.
// Weights (fp16, [tap][Cin/8][CoutPad][8]) are bulk-copied into shared memory once per CTA and stay resident.
#pragma once
#include "ptx.cuh"

namespace dmd {

constexpr int kConvThreads = 384;
constexpr int kConvConsumerWarps = 8;  // warpgroups 1 and 2; each warp releases a ring slot once its wgmma reads retired
constexpr int kTileM = 128;
constexpr int kMaxCin = 128;        // channels of one activation source
constexpr int kMaxSegs = 8;
constexpr int kMaxStages = 24;
constexpr int kStatSlots = 3;   // images a 128-row tile can touch
constexpr int kMaxOutGroups = 4;

struct FastDiv {
  uint32_t d, m;
  __host__ void init(uint32_t dd) {
    d = dd;
    m = (uint32_t)((0x100000000ull / dd) + 1);
  }
  // exact for n*d < 2^32 (host asserts the position count stays below that bound)
  __device__ __forceinline__ uint32_t div(uint32_t n) const { return d == 1 ? n : __umulhi(n, m); }
};

// geometry of a PLC16 tensor over B images of H x W
struct Plc {
  int PW, PH, Q, G, Qalloc;
};
__host__ __device__ inline Plc plc_geometry(int B, int H, int W) {
  Plc g;
  g.PW = W + 1; g.PH = H + 1; g.Q = B * g.PH * g.PW; g.G = g.PW + 1;
  g.Qalloc = g.G + ((g.Q + kTileM - 1) / kTileM) * kTileM + kTileM + g.PW + 1;
  return g;
}

struct ConvParams {
  // K is a concatenation of up to 6 PLC16 operand segments: [x | skip] for a channel concat (blocks.py:174), and
  // [x_hi | skip_hi | x_lo | skip_lo | x_hi | skip_hi] against weights [W_hi | W_hi | W_lo] for split-fp16 convs
  const uint8_t* seg_base[kMaxSegs];
  int seg_slabs[kMaxSegs];  // 16-channel slabs per segment
  int nseg;
  int Cin;              // K channels per tap of the main weights
  int Cextra;           // trailing K channels that use ONLY the centre tap with their own weights: the fused 1x1 skip
                        // projection r = proj(cat(x, skip)) accumulated into the same tile (blocks.py:133,142,145)
  const __half* wpk_extra;  // [1][Cextra/8][CoutPad][8]
  const float* bias_extra;  // [Cout] or null
  int xslabs;               // operand slabs of the projection that are LOADED: hi and lo parts once each (2 * channels / 16)
  int B, H, W;          // conv input size
  int taps;             // 9 (3x3, pad 1) or 1 (1x1)
  int stride;           // 1 or 2 (stride 2 == stride-1 result sampled at even (y,x); exact for k=3,p=1)
  const __half* wpk;    // [taps][Cin/8][CoutPad][8], or [dy][Cin/8][3*CoutPad][8] when trs
  const float* bias;    // [Cout] or null
  int Cout, CoutPad;
  const float* resid;   // NHWC [B][Ho][Wo][Cout] or null
  float* out;           // NHWC [B][Ho][Wo][Cout]
  double* ostats;       // [B][Cout/ogs][2] accumulated with atomics (caller zeroes) or null
  int ogs;
  // derived (host fills)
  int PW, PH, Q, G;
  unsigned long long plane_bytes;  // bytes of one chunk plane (same geometry for both sources)
  int P, Palloc;        // halo positions, odd allocation pitch
  int num_tiles, stages;
  int trs;              // weights in the tap-row-stacked layout (dmd_pack_conv_weight precise = 3): tap (dy, dx) is the column
                        // block dx * CoutPad of kernel row dy
  FastDiv dPW, dPH;
  long long* ktrace;    // diagnostics: globaltimer stamp when the kernel's inputs are ready, or null
};

struct ConvSmemLayout {
  uint32_t bias_off, w_off, a_off, slab_bytes, total;
};

// barriers live in the first 512 bytes: wbar, full[24], empty[24]
__host__ __device__ inline uint32_t conv_weight_bytes(int taps, int Cin, int Cextra, int CoutPad) {
  return (((uint32_t)taps * Cin * CoutPad * 2 + 127u) & ~127u) + (uint32_t)Cextra * CoutPad * 2;
}
// The slab ring follows the weights: a wgmma of N > CoutPad columns (N is a power of two) reads up to N - CoutPad rows past
// the end of a weight block, which stay inside the allocation and only feed accumulator columns that are never stored.
__host__ __device__ inline ConvSmemLayout conv_smem_layout(uint32_t w_bytes, int Palloc, int stages) {
  ConvSmemLayout L;
  L.bias_off = 512;
  L.w_off = L.bias_off + 128 * 4;
  L.a_off = (L.w_off + w_bytes + 127u) & ~127u;
  L.slab_bytes = 2u * Palloc * 16;
  L.total = L.a_off + (uint32_t)stages * L.slab_bytes + 16;
  return L;
}

// ------------------------------------------------------------------------------------------------------------------
// Register epilogue: a consumer thread holds two accumulator rows (r0, r0 + 8) of the tile, columns 8j + 2(lane%4) + {0,1}
// (the wgmma fragment, ptx.cuh): four neighbouring threads hold 32 contiguous bytes of one output row, which go to NHWC global
// memory as full 32-byte sectors (+bias, +residual), with no shared-memory staging.  GroupNorm partial sums run in registers
// across the single-image tiles of a CTA and are reduced with warp shuffles once per image -> fp64 atomics.
template <int N>
struct RegEpilogue {
  int lane, r0, G;
  float s[kStatSlots][kMaxOutGroups], ss[kStatSlots][kMaxOutGroups];
  int n_cur;

  __device__ __forceinline__ void init(const ConvParams& p, int row0, int lane_) {
    lane = lane_;
    r0 = row0;
    G = p.ostats ? p.Cout / p.ogs : 1;
#pragma unroll
    for (int k = 0; k < kStatSlots; ++k)
#pragma unroll
      for (int g = 0; g < kMaxOutGroups; ++g) s[k][g] = ss[k][g] = 0.f;
    n_cur = -1;
  }

  // whole warp, converged.  kG: groups that can hold a nonzero sum (at most kMaxOutGroups).  The butterflies of all groups are
  // independent, so they run round by round side by side instead of one group's five dependent rounds after another's; each
  // value still goes through the same five additions in the same order.
  template <int kG = kMaxOutGroups>
  __device__ __forceinline__ void flush_stats(const ConvParams& p, int img0, int nslots) {
#pragma unroll
    for (int k = 0; k < kStatSlots; ++k) {
      if (k < nslots) {
        float a[kG], b[kG];
#pragma unroll
        for (int g = 0; g < kG; ++g) { a[g] = s[k][g]; b[g] = ss[k][g]; }
#pragma unroll
        for (int m = 16; m > 0; m >>= 1)
#pragma unroll
          for (int g = 0; g < kG; ++g) {
            a[g] += __shfl_xor_sync(0xffffffffu, a[g], m);
            b[g] += __shfl_xor_sync(0xffffffffu, b[g], m);
          }
        if (lane == 0 && img0 + k < p.B) {
#pragma unroll
          for (int g = 0; g < kG; ++g)
            if (g < G && (a[g] != 0.f || b[g] != 0.f)) {
              double* dst = p.ostats + ((size_t)(img0 + k) * G + g) * 2;
              atomicAdd(dst, (double)a[g]);
              atomicAdd(dst + 1, (double)b[g]);
            }
        }
      }
#pragma unroll
      for (int g = 0; g < kMaxOutGroups; ++g) s[k][g] = ss[k][g] = 0.f;
    }
  }

  // the tile starting at padded-linear position q0; acc: this thread's wgmma accumulator fragment.  kLgs: 0 without
  // statistics, else log2 of the 8-column blocks per output group (ogs 16/32/64/128 -> 1..4), so that block j's group j >> kLgs
  // is known at compile time and each block adds straight into its group's sums.  kFull: Cout == N and stride 1 (every
  // stride-1 layer whose Cout is the accumulator width), so every column is stored with an 8-byte access and the column
  // tests and the subsampling compile away; the straight-line code that remains has no branch per column block.
  template <int kLgs, bool kFull>
  __device__ __forceinline__ void tile(const ConvParams& p, const float* sbias, const float (&acc)[N / 2], int q0) {
    constexpr bool kStats = kLgs > 0;
    constexpr int kGroups = (N / 8) >> kLgs > 0 ? ((N / 8) >> kLgs < kMaxOutGroups ? (N / 8) >> kLgs : kMaxOutGroups) : 1;
    const int n_lo = (int)p.dPH.div(p.dPW.div((uint32_t)q0));
    const int q_last = min(q0 + kTileM, p.Q) - 1;
    const bool single_image = (int)p.dPH.div(p.dPW.div((uint32_t)q_last)) == n_lo;
    if (kStats && n_cur >= 0 && (!single_image || n_lo != n_cur)) { flush_stats<kGroups>(p, n_cur, 1); n_cur = -1; }
    const int c0 = 2 * (lane & 3);
    const bool vec = kFull || (p.Cout & 1) == 0;   // 8-byte accesses (every layer but conv_out / the 15-channel dgrad)
    const bool resid = p.resid != nullptr;
    // Every load of a batch (bias from shared memory, residual from global memory) is issued before the batch's first store.
    // The compiler cannot prove that a store to `out` leaves a later load's address alone, so loads placed after stores would
    // each wait out their whole latency in turn.  Up to N = 64 a batch is both rows, all columns: one residual latency per
    // tile instead of one per row, and the bias of a column is read once for both rows.  At N = 128 a batch is 8 column
    // blocks of one row, which bounds the extra registers (that instantiation already uses all 168 a thread can have).
    constexpr int kBatch = N / 8 < 8 ? N / 8 : 8;
    constexpr int kRows = N / 8 <= 8 ? 2 : 1;
#pragma unroll
    for (int h0 = 0; h0 < 2; h0 += kRows) {
      // the output pixel of each row of the batch (-1: a pad position or past the end), and its image slot
      int opix[kRows], slot[kRows];
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const int q = q0 + r0 + 8 * (h0 + r);
        opix[r] = -1; slot[r] = 0;
        if (q < p.Q) {
          const uint32_t R = p.dPW.div((uint32_t)q);
          const int x = q - (int)R * p.PW;
          const int n = (int)p.dPH.div(R);
          const int y = (int)R - n * p.PH;
          bool valid = (x < p.W) && (y < p.H);
          int yo = y, xo = x, Ho = p.H, Wo = p.W;
          if (!kFull && p.stride == 2) {
            valid = valid && ((x & 1) == 0) && ((y & 1) == 0);
            yo = y >> 1; xo = x >> 1; Ho = p.H >> 1; Wo = p.W >> 1;
          }
          if (valid) { opix[r] = (n * Ho + yo) * Wo + xo; slot[r] = n - n_lo; }
        }
      }
      if (kRows == 1 && opix[0] < 0) continue;   // a one-row batch on a pad position: nothing to load, store or count
      float gs[kRows][kMaxOutGroups], gss[kRows][kMaxOutGroups];   // group sums of each row of the batch
#pragma unroll
      for (int r = 0; r < kRows; ++r)
#pragma unroll
        for (int g = 0; g < kMaxOutGroups; ++g) gs[r][g] = gss[r][g] = 0.f;
#pragma unroll
      for (int jb = 0; jb < N / 8; jb += kBatch) {
        float2 bv[kBatch], rv[kRows][kBatch];
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
          const int col = 8 * (jb + u) + c0;
          bv[u] = (kFull || col < p.Cout) ? *reinterpret_cast<const float2*>(sbias + col) : make_float2(0.f, 0.f);
#pragma unroll
          for (int r = 0; r < kRows; ++r) {
            const int h = h0 + r;
            rv[r][u] = make_float2(0.f, 0.f);
            if (resid && opix[r] >= 0 && (kFull || col < p.Cout)) {
              const float* rp = p.resid + (size_t)opix[r] * p.Cout;
              if (vec) rv[r][u] = __ldg(reinterpret_cast<const float2*>(rp + col));
              else {
                rv[r][u].x = __ldg(rp + col);
                if (col + 1 < p.Cout) rv[r][u].y = __ldg(rp + col + 1);
              }
            }
          }
        }
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
          const int h = h0 + r;
          if (opix[r] < 0) continue;
          float* op = p.out + (size_t)opix[r] * p.Cout;
#pragma unroll
          for (int u = 0; u < kBatch; ++u) {
            const int j = jb + u;
            const int col = 8 * j + c0;
            if (kFull || col < p.Cout) {
              float2 o = make_float2(acc[4 * j + 2 * h] + bv[u].x, acc[4 * j + 2 * h + 1] + bv[u].y);
              if (vec) {
                if (resid) { o.x += rv[r][u].x; o.y += rv[r][u].y; }
                *reinterpret_cast<float2*>(op + col) = o;
              } else {
                if (resid) o.x += rv[r][u].x;
                op[col] = o.x;
                if (col + 1 < p.Cout) { if (resid) o.y += rv[r][u].y; op[col + 1] = o.y; } else o.y = 0.f;
              }
              if (kStats) {
                gs[r][j >> kLgs] += o.x + o.y;
                gss[r][j >> kLgs] += fmaf(o.x, o.x, o.y * o.y);
              }
            }
          }
        }
      }
      if (kStats) {
        // Row h's group sums enter the image sums after the row is complete, row 0 before row 1.  Groups and slots that a
        // value does not belong to are skipped rather than given +0.0: every sum starts at +0.0 and so is never -0.0, which
        // makes adding +0.0 an identity, and the sums keep the bits of the select-and-add form.
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
          const int h = h0 + r;
          if (opix[r] < 0) continue;
          if (single_image) {   // warp-uniform: every row of the tile is in image n_lo
#pragma unroll
            for (int g = 0; g < kGroups; ++g) { s[0][g] += gs[r][g]; ss[0][g] += gss[r][g]; }
          } else {
#pragma unroll
            for (int k = 0; k < kStatSlots; ++k)
#pragma unroll
              for (int g = 0; g < kGroups; ++g) {
                s[k][g] += (slot[r] == k) ? gs[r][g] : 0.f;
                ss[k][g] += (slot[r] == k) ? gss[r][g] : 0.f;
              }
          }
        }
      }
    }
    if (kStats) {
      if (single_image) n_cur = n_lo;            // keep running across the single-image tiles of this CTA
      else { flush_stats<kGroups>(p, n_lo, kStatSlots); n_cur = -1; }
    }
  }

  // tile() with the statistics' group size as a template argument (only the sizes an N-column accumulator can hold are
  // instantiated); lgs = log2 of the 8-column blocks per output group, 0 without statistics
  template <bool kFull>
  __device__ __forceinline__ void tile_any(const ConvParams& p, int lgs, const float* sbias, const float (&acc)[N / 2], int q0) {
    if (lgs == 0) tile<0, kFull>(p, sbias, acc, q0);
    else if (lgs == 1 || N == 16) tile<1, kFull>(p, sbias, acc, q0);
    else if (lgs == 2 || N == 32) tile<2, kFull>(p, sbias, acc, q0);
    else if (lgs == 3 || N == 64) tile<3, kFull>(p, sbias, acc, q0);
    else tile<4, kFull>(p, sbias, acc, q0);
  }

  __device__ __forceinline__ void finish(const ConvParams& p) {
    if (p.ostats != nullptr && n_cur >= 0) flush_stats(p, n_cur, 1);
  }
};

// N: accumulator columns (power of two >= CoutPad); kTaps: 9 (3x3) or 1 (1x1), equal to p.taps
template <int N, int kTaps>
__global__ void __launch_bounds__(kConvThreads, 1) conv_tc_kernel(const ConvParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* wbar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* full = wbar + 1;                 // [kMaxStages]
  uint64_t* empty = full + kMaxStages;       // [kMaxStages]
  const ConvSmemLayout L = conv_smem_layout(conv_weight_bytes(p.taps, p.Cin, p.Cextra, p.CoutPad), p.Palloc, p.stages);
  float* sbias = reinterpret_cast<float*>(smem + L.bias_off);
  uint8_t* sW = smem + L.w_off;
  uint8_t* sA = smem + L.a_off;

  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int halo = (kTaps == 9) ? (p.PW + 1) : 0;   // positions in front of the tile's first row
  const int S = p.stages;
  const int main_slabs = p.Cin >> 4;
  const int kslabs = main_slabs + p.xslabs;   // slabs that travel through the ring (the projection's hi slabs feed two MMAs)
  const uint32_t w_main_bytes = ((uint32_t)p.taps * p.Cin * p.CoutPad * 2 + 127u) & ~127u;
  // contiguous, balanced tile range per CTA: neighbouring tiles share halo rows (L2 hits)
  const int tiles_lo = p.num_tiles / (int)gridDim.x, tiles_rem = p.num_tiles % (int)gridDim.x;
  const int tile_begin = (int)blockIdx.x * tiles_lo + min((int)blockIdx.x, tiles_rem);
  const int my_tiles = tiles_lo + ((int)blockIdx.x < tiles_rem ? 1 : 0);

  // ---- setup (independent of the previous kernel: overlaps its tail under programmatic dependent launch)
  pdl_launch_dependents();
  if (tid == 0) {
    mbar_init(wbar, 1);
    for (int s = 0; s < S; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, kConvConsumerWarps); }
    fence_mbar_init();
    const uint32_t tap_bytes = (uint32_t)p.Cin * p.CoutPad * 2;
    const uint32_t extra_bytes = (uint32_t)p.Cextra * p.CoutPad * 2;
    mbar_expect_tx(wbar, tap_bytes * p.taps + extra_bytes);
    for (int t = 0; t < p.taps; ++t)
      bulk_g2s(sW + (size_t)t * tap_bytes, reinterpret_cast<const uint8_t*>(p.wpk) + (size_t)t * tap_bytes, tap_bytes, wbar);
    if (extra_bytes) bulk_g2s(sW + w_main_bytes, p.wpk_extra, extra_bytes, wbar);
  }
  for (int i = tid; i < 128; i += blockDim.x)
    sbias[i] = ((p.bias != nullptr && i < p.Cout) ? __ldg(p.bias + i) : 0.f) + ((p.bias_extra != nullptr && i < p.Cout) ? __ldg(p.bias_extra + i) : 0.f);
  __syncthreads();
  pdl_wait();  // operands / residual / statistics come from earlier kernels
  if (blockIdx.x == 0 && tid == 128) ktrace_stamp(p.ktrace);

  if (warp < 2) {
    // =========================================================================================== PRODUCERS (TMA)
    // Two producer warps take alternate slabs of the global slab sequence: one warp alone spends ~200 cycles per slab (mostly
    // the wait on the `empty` barrier), more than the tensor cores need for the centre-tap slabs of a fused projection.
    // The warp stays converged and one elected lane issues the copies (uniform-register operands).
    const uint32_t pid = (uint32_t)warp;
    const uint32_t chunk_bytes = (uint32_t)p.P * 16;
    uint32_t stage = 0, phase = 0, nslab = 0;
    for (int it = 0; it < my_tiles; ++it) {
      // first halo position of this tile inside a plane (guard G keeps it non-negative)
      const size_t pos0 = (size_t)((tile_begin + it) * kTileM - halo + p.G) * 16;
      int seg = 0, seg_ks = 0;  // current operand segment and slab index inside it
      for (int ks = 0; ks < kslabs; ++ks, ++nslab) {
        if ((nslab & 1u) == pid) {
          mbar_wait(empty + stage, phase ^ 1u);
          if (elect_one_sync()) {
            uint8_t* slab = sA + (size_t)stage * L.slab_bytes;
            // projection slabs (centre tap only): the tile's own 128 rows, no halo
            const bool xs = ks >= main_slabs;
            const uint32_t bytes = xs ? (uint32_t)kTileM * 16 : chunk_bytes;
            mbar_expect_tx(full + stage, 2 * bytes);
            const uint8_t* plane = p.seg_base[seg] + (size_t)(2 * seg_ks) * p.plane_bytes + pos0 + (xs ? (size_t)halo * 16 : 0);
            bulk_g2s(slab, plane, bytes, full + stage);
            bulk_g2s(slab + (size_t)p.Palloc * 16, plane + p.plane_bytes, bytes, full + stage);
          }
          __syncwarp();
        }
        if (++seg_ks == p.seg_slabs[seg]) { seg_ks = 0; ++seg; }
        if (++stage == (uint32_t)S) { stage = 0; phase ^= 1u; }
      }
    }
  } else if (warp >= 4) {
    // =========================================================================================== CONSUMERS (wgmma)
    const int m0 = ((warp >> 2) - 1) * 64;     // first tile row of this warpgroup
    RegEpilogue<N> epi;
    epi.init(p, m0 + 16 * (warp & 3) + (lane >> 2), lane);
    const int lgs = p.ostats ? 31 - __clz(p.ogs >> 3) : 0;   // 8-column block j lies in output group j >> lgs
    const bool full_cols = p.Cout == N && p.stride == 1;      // the epilogue without column tests (RegEpilogue::tile)
    if (my_tiles > 0) mbar_wait(wbar, 0);
    // Descriptor words: per wgmma only the 14-bit start-address fields change (A: ring stage + tap shift, B: tap + slab), all in
    // 16-byte units.  K-major operands: LBO = stride of the 8-channel chunks, SBO = 128 B (eight 16-byte rows).
    const uint64_t hi = gmma_desc_hi(128);
    const uint32_t a_lbo = (uint32_t)p.Palloc * 16;
    const uint32_t b_lbo = (uint32_t)(p.trs ? 3 * p.CoutPad : p.CoutPad) * 16;
    const uint32_t x_lbo = (uint32_t)p.CoutPad * 16;
    const uint32_t a_lo0 = (((smem_u32(sA) + (uint32_t)m0 * 16) >> 4) & 0x3FFFu) | (((a_lbo >> 4) & 0x3FFFu) << 16);
    const uint32_t b_lo0 = ((smem_u32(sW) >> 4) & 0x3FFFu) | (((b_lbo >> 4) & 0x3FFFu) << 16);
    const uint32_t b_x0 = (((smem_u32(sW) + w_main_bytes) >> 4) & 0x3FFFu) | (((x_lbo >> 4) & 0x3FFFu) << 16);
    const uint32_t slab16 = L.slab_bytes >> 4;
    const uint32_t kstep16 = (2u * b_lbo) >> 4;                          // one 16-channel slab of main weights, /16
    const uint32_t xstep16 = (2u * x_lbo) >> 4;                          // one 16-channel slab of projection weights, /16
    uint32_t shift[kTaps], b_tap[kTaps];
#pragma unroll
    for (int t = 0; t < kTaps; ++t) {
      shift[t] = (uint32_t)(halo + (kTaps == 9 ? (t / 3 - 1) * p.PW + (t % 3 - 1) : 0));
      b_tap[t] = p.trs ? ((uint32_t)(t / 3) * p.Cin * 3u * p.CoutPad * 2 + (uint32_t)(t % 3) * p.CoutPad * 16) >> 4
                       : ((uint32_t)t * p.Cin * p.CoutPad * 2) >> 4;
    }
    const int ng = p.xslabs >> 1;   // projection: hi slabs, then as many lo slabs
    float acc[N / 2];
    uint32_t stage = 0, phase = 0, prev = 0;
    int done = 0;                   // slabs of the current tile consumed so far
    // One ring slot: wait for its data, issue the wgmma of `issue` (a fixed, straight-line set: wgmma in a divergent path
    // between fence and commit would make ptxas serialise every wgmma of the kernel), then release the previous slot as soon
    // as its wgmma have retired.
    auto slab = [&](auto issue) {
      mbar_wait(full + stage, phase);
      wgmma_fence();
      issue(a_lo0 + stage * slab16);
      wgmma_commit();
      wgmma_wait<1>();
      if (done > 0 && lane == 0) mbar_arrive(empty + prev);
      prev = stage;
      ++done;
      if (++stage == (uint32_t)S) { stage = 0; phase ^= 1u; }
    };
    for (int it = 0; it < my_tiles; ++it) {
#pragma unroll
      for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
      done = 0;
      for (int ks = 0; ks < main_slabs; ++ks) {
        const uint32_t b_lo = b_lo0 + (uint32_t)ks * kstep16;
        slab([&](uint32_t a_lo) {
#pragma unroll
          for (int t = 0; t < kTaps; ++t) Wgmma<N>::template mma<0, 0>(acc, hi | (a_lo + shift[t]), hi | (b_lo + b_tap[t]), 1u);
        });
      }
      // fused projection (centre tap, slab = the tile's rows): weights [W_hi | W_hi | W_lo] along K; hi slab g meets W_hi
      // (block g) and W_lo (block 2*ng + g), lo slab g meets W_hi (block ng + g)
      for (int g = 0; g < ng; ++g)
        slab([&](uint32_t a_lo) {
          Wgmma<N>::template mma<0, 0>(acc, hi | a_lo, hi | (b_x0 + (uint32_t)g * xstep16), 1u);
          Wgmma<N>::template mma<0, 0>(acc, hi | a_lo, hi | (b_x0 + (uint32_t)(2 * ng + g) * xstep16), 1u);
        });
      for (int g = 0; g < ng; ++g)
        slab([&](uint32_t a_lo) { Wgmma<N>::template mma<0, 0>(acc, hi | a_lo, hi | (b_x0 + (uint32_t)(ng + g) * xstep16), 1u); });
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      if (done > 0 && lane == 0) mbar_arrive(empty + prev);
      const int q0 = (tile_begin + it) * kTileM;
      if (full_cols) epi.template tile_any<true>(p, lgs, sbias, acc, q0);
      else epi.template tile_any<false>(p, lgs, sbias, acc, q0);
    }
    epi.finish(p);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// prep_act_kernel: one pass over an NHWC fp32 tensor that applies what the reference runs on a conv INPUT and writes the
// PLC16 operand:  y = act(a[n][c] * x + b[n][c])  with (a, b) from GroupNorm statistics and FiLM (AdaGroupNorm,
// blocks.py:41-45) or affine weights (blocks.py:28); SiLU (blocks.py:143-144); nearest-2x upsample (blocks.py:109).
// Guard and padding positions are written as zeros, so the buffer needs no memset.
// gridDim.z selects the source (a channel concat is two sources with their own statistics but ONE FiLM vector).
struct PrepSrc {
  const float* src;    // NHWC [B][Hs][Ws][C]
  int C;               // channels stored in src (multiple of 8)
  int Cpad;            // channels of the operand (multiple of 16, >= C; the rest is zero)
  const double* stats; // [B][C/gs][2] or null (mode 0)
  int gs;
  int c_offset;        // channel offset inside the concatenated norm input (FiLM / gamma index = c_offset + c)
  uint8_t* dst;        // PLC16 planes, normalised/activated (fp16 "hi" part)
  uint8_t* dst_lo;     // optional: fp16(y - hi), the low part for split-fp16 convs
  uint8_t* dst_raw;    // optional second output: the raw tensor in PLC16 (for the 1x1 skip projection), or null
  uint8_t* dst_raw_lo; // optional: low part of the raw tensor
};
struct PrepParams {
  PrepSrc s[2];
  int B, Hs, Ws, ups, H, W;   // ups: 0 none, 1 nearest-2x upsample, 2 zero insertion
  int mode;            // 0 raw, 1 AdaGroupNorm, 2 affine GroupNorm
  int act;             // SiLU
  const float* film;   // [B][film_stride]; scale at film_off + c, shift at film_off + film_ctot + c
  int film_stride, film_off, film_ctot;
  const float* gamma;
  const float* beta;
  float eps;
  int PW, PH, Q, G, Qalloc;
  unsigned long long plane_bytes;
  int pos_per_block;
  FastDiv dPW, dPH;
  long long* ktrace;
};

constexpr int kPrepThreads = 256;
constexpr int kPrepBatch = 2;

// low parts of a split-fp16 operand: lo = fp16(v - float(hi))
__device__ __forceinline__ uint4 pack_lo8(const float (&v)[8], const uint4& hi) {
  const __half2* h = reinterpret_cast<const __half2*>(&hi);
  uint4 lo;
  uint32_t* l = reinterpret_cast<uint32_t*>(&lo);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 f = __half22float2(h[k]);
    l[k] = pack_h2(v[2 * k] - f.x, v[2 * k + 1] - f.y);
  }
  return lo;
}

// p.pos_per_block positions per block (multiple of 32, chosen by the host so that a block touches at most 2 images)
__global__ void __launch_bounds__(kPrepThreads, 4) prep_act_kernel(const PrepParams p) {
  __shared__ float sa[2][kMaxCin], sb[2][kMaxCin];  // coefficients for the (at most 2) images this block touches
  __shared__ float smr[2][4][2];                    // (mean, rstd) per (image slot, group)
  pdl_launch_dependents();
  pdl_wait();
  if (blockIdx.x == 0 && blockIdx.z == 0 && threadIdx.x == 0) ktrace_stamp(p.ktrace);
  const PrepSrc& S = p.s[blockIdx.z];
  const int nch = S.Cpad >> 3;
  const int pa0 = blockIdx.x * p.pos_per_block;     // first allocation position of this block
  const int q_first = pa0 - p.G;
  const int n0 = q_first > 0 ? (int)p.dPH.div(p.dPW.div((uint32_t)min(q_first, p.Q - 1))) : 0;
  // lane layout: consecutive lanes = the 8-channel chunks of one pixel (coalesced 32-byte reads of one NHWC row).
  // Items are processed in batches of kPrepBatch with all loads issued first (memory-level parallelism).
  // thread = (chunk j, position lane); it walks positions pl, pl + pstep, ...  (x, y, n) are advanced incrementally, so the
  // per-item cost of locating the source pixel is a few adds instead of two divisions
  const int pstep = kPrepThreads / nch;             // nch in {2, 4, 8, 16}
  const int j = threadIdx.x % nch;
  int pl = threadIdx.x / nch;
  int x, y, n;                                      // coordinates of position pa0 + pl (may be in the guard: q < 0)
  {
    const int q = pa0 + pl - p.G;
    const int qq = q < 0 ? 0 : q;
    const uint32_t R = p.dPW.div((uint32_t)qq);
    x = qq - (int)R * p.PW; n = (int)p.dPH.div(R); y = (int)R - n * p.PH;
    if (q < 0) x += q;                              // negative x marks guard positions until it wraps to >= 0
  }
  const bool has_data = j * 8 < S.C;
  // The first batch of loads does not depend on the coefficients: issue it BEFORE the statistics -> coefficient phase
  // (two barriers and a chain of dependent global loads), whose latency it then hides.
  float4 v0[kPrepBatch], v1[kPrepBatch];
  int meta[kPrepBatch];  // -2: nothing to write, -1: zero fill, else image slot | j << 8
  size_t off[kPrepBatch];
  auto load_batch = [&]() {
#pragma unroll
    for (int u = 0; u < kPrepBatch; ++u) {
      const int pa = pa0 + pl + u * pstep;
      meta[u] = -2;
      if (pl + u * pstep < p.pos_per_block && pa < p.Qalloc) {
        meta[u] = -1;
        off[u] = (size_t)j * p.plane_bytes + (size_t)pa * 16;
        if (has_data && x >= 0 && x < p.W && y < p.H && n < p.B) {
          const int ys = p.ups ? (y >> 1) : y, xs = p.ups ? (x >> 1) : x;
          const float4* gp = reinterpret_cast<const float4*>(S.src + (((size_t)n * p.Hs + ys) * p.Ws + xs) * S.C + j * 8);
          v0[u] = __ldg(gp); v1[u] = __ldg(gp + 1);
          meta[u] = (n - n0) | (j << 8);
        }
      }
      // advance to the next owned position
      x += pstep;
      while (x >= p.PW) { x -= p.PW; if (++y == p.PH) { y = 0; ++n; } }
    }
  };
  load_batch();
  if (p.mode != 0) {
    const int G = S.C / S.gs;
    if (threadIdx.x < 2 * G) {  // fp64 only for the statistics
      const int slot = threadIdx.x / G, g = threadIdx.x - slot * G;
      const int n = n0 + slot;
      float mean_f = 0.f, rstd_f = 0.f;
      if (n < p.B) {
        const double* st = S.stats + ((size_t)n * G + g) * 2;
        const double cnt = (double)p.Hs * p.Ws * S.gs;
        const double mean = st[0] / cnt;
        double var = st[1] / cnt - mean * mean;
        var = var > 0.0 ? var : 0.0;
        mean_f = (float)mean;
        rstd_f = (float)(1.0 / sqrt(var + (double)p.eps));
      }
      smr[slot][g][0] = mean_f;
      smr[slot][g][1] = rstd_f;
    }
    // FiLM / affine loads do not depend on the statistics: issue them before the barrier
    float sc[2] = {0.f, 0.f}, sh[2] = {0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int e = threadIdx.x + k * kPrepThreads;
      if (e < 2 * S.C) {
        const int slot = e / S.C, c = e - slot * S.C;
        const int n = n0 + slot, cg = S.c_offset + c;
        if (n < p.B) {
          if (p.mode == 1) {
            const float* f = p.film + (size_t)n * p.film_stride + p.film_off;
            sc[k] = 1.f + __ldg(f + cg);
            sh[k] = __ldg(f + p.film_ctot + cg);
          } else {
            sc[k] = __ldg(p.gamma + cg);
            sh[k] = __ldg(p.beta + cg);
          }
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int e = threadIdx.x + k * kPrepThreads;
      if (e < 2 * S.C) {
        const int slot = e / S.C, c = e - slot * S.C;
        const float mean = smr[slot][c / S.gs][0], rstd = smr[slot][c / S.gs][1];
        const float a = rstd * sc[k];
        sa[slot][c] = a;
        sb[slot][c] = sh[k] - mean * a;
      }
    }
    __syncthreads();
  }
  for (;;) {
#pragma unroll
    for (int u = 0; u < kPrepBatch; ++u) {
      if (meta[u] == -2) continue;
      uint4 packed = make_uint4(0u, 0u, 0u, 0u), raw = packed, packed_lo = packed, raw_lo = packed;
      if (meta[u] >= 0) {
        const int slot = meta[u] & 0xff, j = meta[u] >> 8;
        float v[8] = {v0[u].x, v0[u].y, v0[u].z, v0[u].w, v1[u].x, v1[u].y, v1[u].z, v1[u].w};
        if (S.dst_raw != nullptr) {
          raw.x = pack_h2(v[0], v[1]); raw.y = pack_h2(v[2], v[3]); raw.z = pack_h2(v[4], v[5]); raw.w = pack_h2(v[6], v[7]);
          if (S.dst_raw_lo != nullptr) raw_lo = pack_lo8(v, raw);
        }
        if (p.mode != 0) {
          const float4* ca = reinterpret_cast<const float4*>(&sa[slot][j * 8]);
          const float4* cb = reinterpret_cast<const float4*>(&sb[slot][j * 8]);
          const float4 a0 = ca[0], a1 = ca[1], b0 = cb[0], b1 = cb[1];
          v[0] = fmaf(a0.x, v[0], b0.x); v[1] = fmaf(a0.y, v[1], b0.y); v[2] = fmaf(a0.z, v[2], b0.z); v[3] = fmaf(a0.w, v[3], b0.w);
          v[4] = fmaf(a1.x, v[4], b1.x); v[5] = fmaf(a1.y, v[5], b1.y); v[6] = fmaf(a1.z, v[6], b1.z); v[7] = fmaf(a1.w, v[7], b1.w);
        }
        if (p.act) {
#pragma unroll
          for (int k = 0; k < 8; ++k) v[k] = silu_f(v[k]);
        }
        packed.x = pack_h2(v[0], v[1]); packed.y = pack_h2(v[2], v[3]); packed.z = pack_h2(v[4], v[5]); packed.w = pack_h2(v[6], v[7]);
        if (S.dst_lo != nullptr) packed_lo = pack_lo8(v, packed);
      }
      *reinterpret_cast<uint4*>(S.dst + off[u]) = packed;
      if (S.dst_lo != nullptr) *reinterpret_cast<uint4*>(S.dst_lo + off[u]) = packed_lo;
      if (S.dst_raw != nullptr) *reinterpret_cast<uint4*>(S.dst_raw + off[u]) = raw;
      if (S.dst_raw_lo != nullptr) *reinterpret_cast<uint4*>(S.dst_raw_lo + off[u]) = raw_lo;
    }
    pl += kPrepBatch * pstep;
    if (pl >= p.pos_per_block) break;
    load_batch();
  }
}

// prep_fast_kernel: the hot cases of prep_act_kernel with everything else compiled out -- GroupNorm / AdaGroupNorm + SiLU, no
// upsample, no low part of the normalised operand; RAW additionally emits the raw operand and its low part (the split-fp16
// operand of the fused 1x1 skip projection).  prep_act_kernel executes ~225 instructions per 8-channel item (ncu: 7.6 M
// warp-instructions per 64x64x64-channel launch, issue-bound), most of them generic-path bookkeeping: here the chunk count is a
// template parameter, a thread owns ONE 8-channel chunk and walks positions, addresses are 32-bit, and four items are in flight
// per thread.  Same grid, same PrepParams, bit-identical results.
template <int NCH, bool RAW>
__global__ void __launch_bounds__(kPrepThreads, 4) prep_fast_kernel(const PrepParams p) {
  __shared__ float sa[2][kMaxCin], sb[2][kMaxCin];  // coefficients for the (at most 2) images this block touches
  __shared__ float smr[2][4][2];                    // (mean, rstd) per (image slot, group)
  constexpr int PSTEP = kPrepThreads / NCH;
  constexpr int kBatch = 4;
  pdl_launch_dependents();
  pdl_wait();
  if (blockIdx.x == 0 && blockIdx.z == 0 && threadIdx.x == 0) ktrace_stamp(p.ktrace);
  const PrepSrc& S = p.s[blockIdx.z];
  const int pa0 = blockIdx.x * p.pos_per_block;     // first allocation position of this block
  const int q_first = pa0 - p.G;
  const int n0 = q_first > 0 ? (int)p.dPH.div(p.dPW.div((uint32_t)min(q_first, p.Q - 1))) : 0;
  const int j = threadIdx.x & (NCH - 1);
  int pl = threadIdx.x / NCH;
  int x, y, n;                                      // coordinates of position pa0 + pl (x < 0: still inside the front guard)
  {
    const int q = pa0 + pl - p.G;
    const int qq = q < 0 ? 0 : q;
    const uint32_t R = p.dPW.div((uint32_t)qq);
    x = qq - (int)R * p.PW; n = (int)p.dPH.div(R); y = (int)R - n * p.PH;
    if (q < 0) x += q;
  }
  const bool has_data = j * 8 < S.C;
  // ---- statistics -> coefficients (identical to prep_act_kernel)
  {
    const int G = S.C / S.gs;
    if (threadIdx.x < 2 * G) {
      const int slot = threadIdx.x / G, g = threadIdx.x - slot * G;
      const int ni = n0 + slot;
      float mean_f = 0.f, rstd_f = 0.f;
      if (ni < p.B) {
        const double* st = S.stats + ((size_t)ni * G + g) * 2;
        const double cnt = (double)p.Hs * p.Ws * S.gs;
        const double mean = st[0] / cnt;
        double var = st[1] / cnt - mean * mean;
        var = var > 0.0 ? var : 0.0;
        mean_f = (float)mean;
        rstd_f = (float)(1.0 / sqrt(var + (double)p.eps));
      }
      smr[slot][g][0] = mean_f;
      smr[slot][g][1] = rstd_f;
    }
    float sc[2] = {0.f, 0.f}, sh[2] = {0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int e = threadIdx.x + k * kPrepThreads;
      if (e < 2 * S.C) {
        const int slot = e / S.C, c = e - slot * S.C;
        const int ni = n0 + slot, cg = S.c_offset + c;
        if (ni < p.B) {
          if (p.mode == 1) {
            const float* f = p.film + (size_t)ni * p.film_stride + p.film_off;
            sc[k] = 1.f + __ldg(f + cg);
            sh[k] = __ldg(f + p.film_ctot + cg);
          } else {
            sc[k] = __ldg(p.gamma + cg);
            sh[k] = __ldg(p.beta + cg);
          }
        }
      }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int e = threadIdx.x + k * kPrepThreads;
      if (e < 2 * S.C) {
        const int slot = e / S.C, c = e - slot * S.C;
        const float mean = smr[slot][c / S.gs][0], rstd = smr[slot][c / S.gs][1];
        const float a = rstd * sc[k];
        sa[slot][c] = a;
        sb[slot][c] = sh[k] - mean * a;
      }
    }
    __syncthreads();
  }
  uint8_t* const d_n = S.dst + (size_t)j * p.plane_bytes + (size_t)pa0 * 16;
  uint8_t* const d_r = RAW ? S.dst_raw + (size_t)j * p.plane_bytes + (size_t)pa0 * 16 : nullptr;
  uint8_t* const d_rl = RAW ? S.dst_raw_lo + (size_t)j * p.plane_bytes + (size_t)pa0 * 16 : nullptr;
  const int limit = min(p.pos_per_block, p.Qalloc - pa0);   // positions this block writes
  const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
  for (; pl < limit; pl += kBatch * PSTEP) {
    float4 v0[kBatch], v1[kBatch];
    int slot[kBatch];                                // -1: zero fill
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      slot[u] = -1;
      if (pl + u * PSTEP < limit && has_data && x >= 0 && x < p.W && y < p.H && n < p.B) {
        const uint32_t idx = (uint32_t)((n * p.Hs + y) * p.Ws + x) * (uint32_t)S.C + (uint32_t)(j * 8);
        const float4* gp = reinterpret_cast<const float4*>(S.src + idx);
        v0[u] = __ldg(gp); v1[u] = __ldg(gp + 1);
        slot[u] = n - n0;
      }
      x += PSTEP;
      while (x >= p.PW) { x -= p.PW; if (++y == p.PH) { y = 0; ++n; } }
    }
#pragma unroll
    for (int u = 0; u < kBatch; ++u) {
      const int pp = pl + u * PSTEP;
      if (pp >= limit) break;
      uint4 packed = zero4, raw = zero4, raw_lo = zero4;
      if (slot[u] >= 0) {
        const float4* pa4 = reinterpret_cast<const float4*>(&sa[slot[u]][j * 8]);
        const float4* pb4 = reinterpret_cast<const float4*>(&sb[slot[u]][j * 8]);
        const float4 a0 = pa4[0], a1 = pa4[1], b0 = pb4[0], b1 = pb4[1];
        const float ca[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float cb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
        float v[8] = {v0[u].x, v0[u].y, v0[u].z, v0[u].w, v1[u].x, v1[u].y, v1[u].z, v1[u].w};
        if (RAW) {
          raw.x = pack_h2(v[0], v[1]); raw.y = pack_h2(v[2], v[3]); raw.z = pack_h2(v[4], v[5]); raw.w = pack_h2(v[6], v[7]);
          raw_lo = pack_lo8(v, raw);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) v[k] = silu_f(fmaf(ca[k], v[k], cb[k]));
        packed.x = pack_h2(v[0], v[1]); packed.y = pack_h2(v[2], v[3]); packed.z = pack_h2(v[4], v[5]); packed.w = pack_h2(v[6], v[7]);
      }
      *reinterpret_cast<uint4*>(d_n + (size_t)pp * 16) = packed;
      if (RAW) {
        *reinterpret_cast<uint4*>(d_r + (size_t)pp * 16) = raw;
        *reinterpret_cast<uint4*>(d_rl + (size_t)pp * 16) = raw_lo;
      }
    }
  }
}

// Zero-insertion operand (ups == 2): the adjoint of the stride-2 subsample of Downsample (blocks.py:96).  src is the NHWC
// fp32 gradient at the conv OUTPUT size [B][Hs][Ws][C]; the PLC16 operand at the conv INPUT size (2Hs x 2Ws) carries it at the
// even (y, x) and zeros everywhere else.  One thread per (position, 8-channel chunk).  (A separate kernel on purpose: adding
// this case to prep_act_kernel's load predicate made ptxas 12.9 emit a kernel whose coefficient phase went stale.)
__global__ void __launch_bounds__(256) zero_insert_prep_kernel(const PrepParams p) {
  pdl_launch_dependents();
  pdl_wait();
  const PrepSrc& S = p.s[0];
  const int nch = S.Cpad >> 3;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)p.Qalloc * nch;
  if (idx >= total) return;
  const int j = (int)(idx % nch);
  const int pa = (int)(idx / nch);
  uint4 packed = make_uint4(0u, 0u, 0u, 0u);
  const int q = pa - p.G;
  if (q >= 0 && q < p.Q && j * 8 < S.C) {
    const uint32_t R = p.dPW.div((uint32_t)q);
    const int x = q - (int)R * p.PW;
    const int n = (int)p.dPH.div(R);
    const int y = (int)R - n * p.PH;
    if (x < p.W && y < p.H && ((x | y) & 1) == 0) {
      const float4* gp = reinterpret_cast<const float4*>(S.src + (((size_t)n * p.Hs + (y >> 1)) * p.Ws + (x >> 1)) * S.C + j * 8);
      const float4 a = __ldg(gp), b = __ldg(gp + 1);
      packed.x = pack_h2(a.x, a.y); packed.y = pack_h2(a.z, a.w); packed.z = pack_h2(b.x, b.y); packed.w = pack_h2(b.z, b.w);
    }
  }
  *reinterpret_cast<uint4*>(S.dst + (size_t)j * p.plane_bytes + (size_t)pa * 16) = packed;
}

}  // namespace dmd
