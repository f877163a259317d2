// Weight gradient of the 3x3 / 1x1 convolutions on Hopper tensor cores (sm_90a wgmma).
//
// Backward-filter of nn.Conv2d (reference: blocks.py:18-19,96,109-110; torch autograd's conv2d_weight):
//     dW[co][ci][t] = sum over positions q of  GY[q][co] * X[q + o_t][ci],      o_t = (ky-1)*PW + (kx-1)
// on the SAME padded-linear PLC16 operands the forward kernel reads (conv_tc.cuh): positions are the GEMM K dimension, and
// a PLC16 chunk plane -- 16 bytes (8 channels) per position, positions contiguous -- is exactly the wgmma no-swizzle
// MN-MAJOR canonical layout (core matrix = 8 positions x 16 B).  Out-of-image taps read the shared zero pads and GY is zero
// at pad positions, so there are NO boundary tests (oracle/backward_plan.py wgrad_over_positions pins this formulation).
//
//   A (M = 64 rows = output channels) = the gradient operand of a 128-position tile, eight chunk planes (zeros beyond Cg).
//   B (N = Cin <= 64) = the activation operand with a PW+1 halo; tap t shifts the descriptor start address by o_t * 16 B.
//   D: nine fp32 accumulators, one per tap, in registers and alive across ALL tiles of the CTA; one epilogue at the end
//      writes the CTA's partial sums, and wgrad_reduce_kernel adds the partials in a fixed order (deterministic split-K) into
//      the torch-layout gradient.
//
// Roles (416 threads, one CTA per SM, contiguous tile range): warpgroup c = 0, 1, 2 owns kernel row ky = c (three taps, three
// m64 x N accumulators: 3 * N / 2 registers per thread); warp 12 is the producer (cp.async.bulk, 8 + nB copies per tile).
#pragma once
#include <type_traits>
#include "conv_tc.cuh"

namespace dmd {

constexpr int kWgThreads = 416;
constexpr int kWgConsumerWarps = 12;
constexpr int kWgTaps = 9;
constexpr int kWgStagesMax = 4;

struct WgradParams {
  const uint8_t* a_plane[8];    // gradient chunk plane feeding rows 8g .. 8g+7; null = all-zero rows
  const uint8_t* zeros;         // >= 2 KB of zeros (source of the null groups)
  const uint8_t* b_plane[8];    // activation chunk planes (N = 8 * nB channels)
  int nB;
  int taps;                     // 9 or 1
  int PW;
  int halo;                     // PW + 1 (3x3) or 0
  int G;                        // guard positions in front of position 0 of every plane
  int num_tiles, stages;
  int Pb;                       // activation positions per stage (128 + 2*halo), PbAlloc = Pb | 1
  float* partial;               // [gridDim.x][taps][64][N]
};

struct WgradSmem { uint32_t a_off, b_off, a_bytes, b_bytes, total; };
__host__ __device__ inline WgradSmem wgrad_smem(int nB, int halo, int stages) {
  WgradSmem L;
  const uint32_t PbAlloc = (uint32_t)((kTileM + 2 * halo) | 1);
  L.a_bytes = 8u * kTileM * 16u;                  // 16 KB: 8 row groups x 128 positions x 16 B
  L.b_bytes = ((uint32_t)nB * PbAlloc * 16u + 127u) & ~127u;
  L.a_off = 256;                                  // barriers first
  L.b_off = L.a_off + (uint32_t)stages * L.a_bytes;
  L.total = L.b_off + (uint32_t)stages * L.b_bytes + 16;
  return L;
}

template <int N>
__global__ void __launch_bounds__(kWgThreads, 1) wgrad_tc_kernel(const WgradParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);   // [kWgStagesMax]
  uint64_t* empty = full + kWgStagesMax;                // [kWgStagesMax]
  const WgradSmem L = wgrad_smem(p.nB, p.halo, p.stages);
  uint8_t* sA = smem + L.a_off;
  uint8_t* sB = smem + L.b_off;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int S = p.stages;
  const uint32_t PbAlloc = (uint32_t)(p.Pb | 1);
  const int tiles_lo = p.num_tiles / (int)gridDim.x, tiles_rem = p.num_tiles % (int)gridDim.x;
  const int tile_begin = (int)blockIdx.x * tiles_lo + min((int)blockIdx.x, tiles_rem);
  const int my_tiles = tiles_lo + ((int)blockIdx.x < tiles_rem ? 1 : 0);

  pdl_launch_dependents();
  if (tid == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(full + s, 1); mbar_init(empty + s, kWgConsumerWarps); }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();

  if (warp == kWgConsumerWarps) {
    // ================================================================================================= PRODUCER
    uint32_t stage = 0, phase = 0;
    const uint32_t b_chunk = (uint32_t)p.Pb * 16;
    for (int it = 0; it < my_tiles; ++it) {
      const long long q0 = (long long)(tile_begin + it) * kTileM;
      mbar_wait(empty + stage, phase ^ 1u);
      if (elect_one_sync()) {
        mbar_expect_tx(full + stage, 8u * kTileM * 16u + (uint32_t)p.nB * b_chunk);
        uint8_t* a = sA + (size_t)stage * L.a_bytes;
#pragma unroll 1
        for (int g = 0; g < 8; ++g)
          bulk_g2s(a + (size_t)g * (kTileM * 16), p.a_plane[g] ? p.a_plane[g] + (size_t)(p.G + q0) * 16 : p.zeros, kTileM * 16, full + stage);
        uint8_t* b = sB + (size_t)stage * L.b_bytes;
#pragma unroll 1
        for (int j = 0; j < p.nB; ++j)
          bulk_g2s(b + (size_t)j * PbAlloc * 16, p.b_plane[j] + (size_t)(p.G + q0 - p.halo) * 16, b_chunk, full + stage);
      }
      __syncwarp();
      if (++stage == (uint32_t)S) { stage = 0; phase ^= 1u; }
    }
  } else {
    // ================================================================================================= CONSUMERS
    const int ky = warp >> 2;                 // kernel row of this warpgroup
    const int ntap = p.taps == 9 ? 3 : (ky == 0 ? 1 : 0);
    // MN-major no-swizzle: K groups (8 positions) are 128 B apart; MN groups (8 channels) one plane apart
    const uint32_t a_lbo = 128, a_sbo = kTileM * 16, b_lbo = 128, b_sbo = PbAlloc * 16;
    const uint64_t a_hi = gmma_desc_hi(a_sbo), b_hi = gmma_desc_hi(b_sbo);
    const uint32_t a_lo0 = ((smem_u32(sA) >> 4) & 0x3FFFu) | (((a_lbo >> 4) & 0x3FFFu) << 16);
    const uint32_t b_lo0 = ((smem_u32(sB) >> 4) & 0x3FFFu) | (((b_lbo >> 4) & 0x3FFFu) << 16);
    uint32_t bsh[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) bsh[i] = (uint32_t)(p.halo + (p.taps == 9 ? (ky - 1) * p.PW + (i - 1) : 0));
    float acc[3][N / 2];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int k = 0; k < N / 2; ++k) acc[i][k] = 0.f;
    uint32_t stage = 0, phase = 0, prev = 0;
    for (int it = 0; it < my_tiles; ++it) {
      mbar_wait(full + stage, phase);
      if (ntap > 0) {
        wgmma_fence();
        const uint32_t a_st = a_lo0 + stage * (L.a_bytes >> 4), b_st = b_lo0 + stage * (L.b_bytes >> 4);
        // the tap count is a compile-time constant inside the loop: no predicated wgmma between the fence and the commit
        auto mma_tile = [&](auto ntc) {
          constexpr int NT = decltype(ntc)::value;
#pragma unroll
          for (int ks = 0; ks < kTileM / 16; ++ks) {
            const uint64_t ad = a_hi | (a_st + (uint32_t)ks * 16u);
#pragma unroll
            for (int i = 0; i < NT; ++i) Wgmma<N>::template mma<1, 1>(acc[i], ad, b_hi | (b_st + bsh[i] + (uint32_t)ks * 16u), 1u);
          }
        };
        if (ntap == 3) mma_tile(std::integral_constant<int, 3>{});
        else mma_tile(std::integral_constant<int, 1>{});
        wgmma_commit();
        wgmma_wait<1>();                     // the previous tile's wgmma have retired: its ring slot is free
      }
      if (it > 0 && lane == 0) mbar_arrive(empty + prev);
      prev = stage;
      if (++stage == (uint32_t)S) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 3; ++i) wgmma_fence_operands(acc[i]);
    // partials [taps][64][N]: rows r, r + 8 of the fragment, columns 8j + 2(lane%4) + {0,1}
    const int r = 16 * (warp & 3) + (lane >> 2), c = 2 * (lane & 3);
    float* out = p.partial + (size_t)blockIdx.x * p.taps * 64 * N;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      if (i < ntap) {
        float* o = out + (size_t)(3 * ky + i) * 64 * N;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) {
          *reinterpret_cast<float2*>(o + (size_t)r * N + 8 * j + c) = make_float2(acc[i][4 * j], acc[i][4 * j + 1]);
          *reinterpret_cast<float2*>(o + (size_t)(r + 8) * N + 8 * j + c) = make_float2(acc[i][4 * j + 2], acc[i][4 * j + 3]);
        }
      }
    }
  }
}

// Fixed-order reduction of the per-CTA partials into the torch-layout weight gradient [Cout][CinTot][taps] (fp32):
//   dW[co][ci_off + ci][t] (+)= inv_scale * sum_part partial[part][t][co][ci]
// inv_scale undoes the loss scaling of the gradient operand (device scalar).
struct WgradReduceParams {
  const float* partial; int nparts; int N;
  float* dW; int Cout, Cin, CinTot, ci_off, taps;
  int co_off;                   // first output channel (row of dW) of this launch's 64-row block
  const float* inv_scale;       // device scalar or null (1.0)
  int accumulate;
};
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const WgradReduceParams p) {
  // 64 consecutive outputs per block x 4 groups of partials: thread (kg, o) adds partials kg, kg + 4, ... of output o with four
  // independent accumulators (the loads of one output are one CTA partial block apart: latency-bound unless many are in flight),
  // then the four groups are combined through shared memory.  The order of every addition is fixed, so the result is deterministic.
  __shared__ float part[4][64];
  const int o = threadIdx.x & 63, kg = threadIdx.x >> 6;
  const int idx = blockIdx.x * 64 + o;        // == offset of the element inside one CTA's partial block [taps][64][N]
  const int per = 64 * p.N;
  int t = -1, co = 0, ci = 0;
  if (idx < p.taps * per) {
    t = idx / per;
    const int r = idx - t * per;
    co = r / p.N;
    ci = r - co * p.N;
  }
  const bool live = t >= 0 && co < p.Cout && ci < p.Cin;
  float s = 0.f;
  if (live) {
    const size_t stride = (size_t)p.taps * per;
    const float* src = p.partial + idx;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int k = kg;
    for (; k + 12 < p.nparts; k += 16) {
      a0 += src[(size_t)k * stride]; a1 += src[(size_t)(k + 4) * stride];
      a2 += src[(size_t)(k + 8) * stride]; a3 += src[(size_t)(k + 12) * stride];
    }
    for (; k < p.nparts; k += 4) a0 += src[(size_t)k * stride];
    s = (a0 + a1) + (a2 + a3);
  }
  part[kg][o] = s;
  __syncthreads();
  if (kg == 0 && live) {
    s = (part[0][o] + part[1][o]) + (part[2][o] + part[3][o]);
    if (p.inv_scale) s *= *p.inv_scale;
    float* d = p.dW + ((size_t)(p.co_off + co) * p.CinTot + p.ci_off + ci) * p.taps + t;
    *d = p.accumulate ? *d + s : s;
  }
}

}  // namespace dmd
