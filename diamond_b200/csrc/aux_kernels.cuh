// Small CUDA-core kernels around the tensor-core convolution: everything on the denoiser path that is not a conv.
// Each kernel cites the reference lines it replaces.  No fast-math: sqrt / div are IEEE so the EDM conditioners and
// the uint8 quantiser reproduce the reference's fp32 arithmetic bit for bit where it matters (denoiser.py:66-84).
#pragma once
#include <cooperative_groups.h>
#include <type_traits>
#include "ptx.cuh"

namespace dmd {

// ------------------------------------------------------------------------------------------------
// EDM conditioners (denoiser.py:66-72).  cs[n] = {c_in, c_out, c_skip, c_noise}
__device__ __forceinline__ float4 edm_conditioners(float sigma, float sigma_data, float sigma_offset) {
  const float s2 = __fadd_rn(__fmul_rn(sigma, sigma), __fmul_rn(sigma_offset, sigma_offset));
  const float s = __fsqrt_rn(s2);
  const float sd2 = __fmul_rn(sigma_data, sigma_data);
  const float den = __fadd_rn(__fmul_rn(s, s), sd2);
  float4 c;
  c.x = __fdiv_rn(1.0f, __fsqrt_rn(den));  // c_in
  c.z = __fdiv_rn(sd2, den);               // c_skip
  c.y = __fmul_rn(s, __fsqrt_rn(c.z));     // c_out
  c.w = __fdiv_rn(logf(s), 4.0f);          // c_noise
  return c;
}

// Where the frame stack / action stack of the sampler lives.  Default (ring_T = 0): obs (B, T*C, H, W), act (B, T) as the
// reference passes them.  Ring (ring_T = T): the WorldModelEnv's resident buffers frames (T, B, C, H, W) / acts (T, B), where
// LOGICAL slot k (0 = oldest) is physical slot (head + k) % T -- the reference's per-step `roll` of both buffers
// (world_model_env.py:74-75) becomes head = (head + 1) % T and no data moves.
struct StackView { int ring_T; int head; long long frame_stride; long long batch_stride; long long act_slot_stride; long long act_batch_stride; };

// Frames stored as one byte per value (dmd_u8_frames, include/diamond_b200.h).  Value (n, f, i) -- sample n, frame f, element
// i = channel * H*W + pixel -- is table[kind * 256 + byte] with byte = levels[n * batch_stride + f * frame_stride + i] and
// kind = kinds[n * kind_batch_stride + f * kind_frame_stride]: the table holds, per kind, the fp32 value an fp32 frame source
// would hold for that byte (diamond_b200/frames.py builds it), so a decoded frame is bit-identical to the fp32 one.  A kind
// outside [0, kFrameKinds) decodes as kind 0 (padding).
constexpr int kFrameKinds = 3;
struct U8Frames {
  const uint8_t* levels; long long batch_stride; long long frame_stride;
  const uint8_t* kinds; long long kind_batch_stride; long long kind_frame_stride;
  const float* table;
};
// the decode table in shared memory; every thread of the block must call it (it synchronises)
__device__ __forceinline__ const float* stage_decode_table(const float* __restrict__ table) {
  __shared__ float tab[kFrameKinds * 256];
  for (int i = threadIdx.x; i < kFrameKinds * 256; i += blockDim.x) tab[i] = table[i];
  __syncthreads();
  return tab;
}
__device__ __forceinline__ float u8_frame_value(const U8Frames& s, const float* tab, long long n, long long f, size_t i) {
  unsigned kind = s.kinds[(size_t)n * s.kind_batch_stride + (size_t)f * s.kind_frame_stride];
  if (kind >= (unsigned)kFrameKinds) kind = 0;
  return tab[kind * 256 + s.levels[(size_t)n * s.batch_stride + (size_t)f * s.frame_stride + i]];
}

// Pack the conv_in input (inner_model.py:46 cat((obs, noisy)) after denoiser.py:75-76 rescaling) as NHWC with the
// channel count rounded up to CP (multiple of 8; zero filled).   obs: (B, Cobs, H, W) fp32 (Obs = const float*), or the
// Cobs / Cimg frames of a U8Frames source (Obs = U8Frames; sv is not used);  noisy: (B, Cimg, H, W) NCHW.
// Also writes cs[n] (4 floats).  grid: (ceil(H*W/256), B)
template <class Obs>
__global__ void pack_denoiser_input_kernel(const float* __restrict__ noisy, const Obs obs,
                                           const float* __restrict__ sigma, int sigma_is_scalar, float* __restrict__ xin,
                                           float* __restrict__ cs, int Cobs, int Cimg, int CP, int HW, float sigma_data,
                                           float sigma_offset, int prescaled, StackView sv) {
  constexpr bool kU8 = std::is_same<Obs, U8Frames>::value;
  [[maybe_unused]] const float* tab = nullptr;
  if constexpr (kU8) tab = stage_decode_table(obs.table);
  const int n = blockIdx.y;
  const float sg = sigma[sigma_is_scalar ? 0 : n];
  // prescaled: caller already applied denoiser.py:75-76 and `sigma` holds c_noise (InnerModel.forward surface)
  const float4 c = prescaled ? make_float4(1.f, 0.f, 0.f, sg) : edm_conditioners(sg, sigma_data, sigma_offset);
  if (blockIdx.x == 0 && threadIdx.x == 0) reinterpret_cast<float4*>(cs)[n] = c;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= HW) return;
  float* o = xin + ((size_t)n * HW + pix) * CP;
  for (int ch = 0; ch < CP; ++ch) {
    float v = 0.f;
    if (ch < Cobs) {
      if constexpr (kU8) {
        const int f = ch / Cimg, cc = ch - f * Cimg;
        v = u8_frame_value(obs, tab, n, f, (size_t)cc * HW + pix);
      } else if (sv.ring_T > 0) {
        const int f = ch / Cimg, cc = ch - f * Cimg;
        int pf = sv.head + f; if (pf >= sv.ring_T) pf -= sv.ring_T;
        v = obs[(size_t)pf * sv.frame_stride + (size_t)n * sv.batch_stride + (size_t)cc * HW + pix];
      } else {
        v = obs[((size_t)n * Cobs + ch) * HW + pix];
      }
      if (!prescaled) v = __fdiv_rn(v, sigma_data);
    } else if (ch < Cobs + Cimg) {
      v = __fmul_rn(noisy[((size_t)n * Cimg + (ch - Cobs)) * HW + pix], c.x);
    }
    o[ch] = v;
  }
}

// Generic NCHW -> NHWC(+channel pad) and back, fp32 (actor-critic observations, tests).
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int CP, int HW) {
  const int n = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= HW) return;
  float* o = out + ((size_t)n * HW + pix) * CP;
  for (int ch = 0; ch < CP; ++ch) o[ch] = ch < C ? in[((size_t)n * C + ch) * HW + pix] : 0.f;
}
__global__ void nhwc_to_nchw_kernel(const float* __restrict__ in, float* __restrict__ out, int C, int CP, int HW) {
  const int n = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= HW) return;
  const float* i = in + ((size_t)n * HW + pix) * CP;
  for (int ch = 0; ch < C; ++ch) out[((size_t)n * C + ch) * HW + pix] = i[ch];
}

// Zero-pad / crop of an NHWC fp32 tensor at the bottom / right edges (UNet.forward, blocks.py:225-229 `F.pad(x, (0, pw, 0, ph))` and
// :245 `x[..., :h, :w]`): dst[n][y][x][:] = (y < Hs && x < Ws) ? src[n][y][x][:] : 0.  One float4 per thread; C % 4 == 0.
struct ResizeParams { const float* src; float* dst; int B, Hs, Ws, Hd, Wd, C; double* stats; int gs; };
__global__ void resize_nhwc_kernel(const ResizeParams p) {
  const int C4 = p.C >> 2;
  const long long total = (long long)p.B * p.Hd * p.Wd * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c4 = (int)(i % C4);
    long long r = i / C4;
    const int x = (int)(r % p.Wd); r /= p.Wd;
    const int y = (int)(r % p.Hd);
    const int n = (int)(r / p.Hd);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (y < p.Hs && x < p.Ws) v = __ldg(reinterpret_cast<const float4*>(p.src + (((size_t)n * p.Hs + y) * p.Ws + x) * p.C) + c4);
    reinterpret_cast<float4*>(p.dst)[i] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// Conditioning path (inner_model.py:45, :27-35; blocks.py:84-87, :39,44), as one embedding kernel + three calls of a
// small GEMM:   e = fourier(c_noise) + flatten(act_emb(act)) ;  h = silu(W0 e + b0) ;  cond = W1 h + b1 ;
//               film = Wf cond + bf   (ALL AdaGroupNorm linears of the network batched: Wf = [sum 2C][CC])
// cs != null: c_noise of sample n is cs[n][3] (written by the pack kernel).  cs == null: row r = (evaluation k, sample n) of a
// batch of K sampler evaluations, c_noise computed from sig_all[k] (all denoising steps' conditioning in ONE launch: the sigma
// schedule is host-known, diffusion_sampler.py:27, and the actions do not change inside sample()).
__global__ void cond_embed_kernel(const float* __restrict__ cs, const float* __restrict__ sig_all, float sigma_data, float sigma_offset,
                                  const int64_t* __restrict__ act, const float* __restrict__ fourier_w, const float* __restrict__ act_emb,
                                  float* __restrict__ e, int rows, int B, int CC, int T, int num_actions, StackView sv) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * CC) return;
  const int r = i / CC, k = i - r * CC;
  const int n = r % B;
  const int half = CC / 2, E = CC / T;
  const float c_noise = cs ? cs[n * 4 + 3] : edm_conditioners(sig_all[r / B], sigma_data, sigma_offset).w;
  const float t = __fmul_rn(6.283185307179586f, c_noise);
  const float f = __fmul_rn(t, fourier_w[k < half ? k : k - half]);
  const float four = k < half ? cosf(f) : sinf(f);
  long long a;
  if (sv.ring_T > 0) {
    int ps = sv.head + k / E; if (ps >= sv.ring_T) ps -= sv.ring_T;
    a = act[(size_t)ps * sv.act_slot_stride + (size_t)n * sv.act_batch_stride];
  } else {
    a = act[(size_t)n * T + k / E];
  }
  a = a < 0 ? 0 : (a >= num_actions ? num_actions - 1 : a);
  e[i] = __fadd_rn(four, act_emb[(size_t)a * E + (k % E)]);
}

// out[n][f] (+)= act( sum_k in[n][k] * W[f][k] + b[f] ),  K multiple of 4; K is processed in chunks of <= 256.
// grid (ceil(F/(8J)), ceil(B/32)), 256 threads: warp w owns rows f = Jw..Jw+J-1 of the 8J-row tile, lane = sample n.
// J = 1 gives small GEMMs (the conditioning MLP: F = cond_channels, 32..2048) four times the blocks; the k order of each sum is
// the same.  Any K and F are covered (K in chunks of kLinChunk, F in tiles of 8J rows); linear_launch picks J from the grid size.
// hw_perm > 0: `in` is an NHWC tensor [B][hw_perm][K/hw_perm] read in NCHW-flatten order (k = c*hw + pix), i.e. the
// x.flatten(start_dim=1) of actor_critic.py:71 without materialising the permutation.
constexpr int kLinChunk = 256;
template <int J>
__global__ void __launch_bounds__(256) linear_kernel(const float* __restrict__ in, const float* __restrict__ W,
                                                     const float* __restrict__ bias, float* __restrict__ out, int B,
                                                     int K, int F, int silu, int accumulate, int hw_perm) {
  extern __shared__ __align__(16) float sm_lin[];
  constexpr int FT = 8 * J;              // output features per block
  float* Ws = sm_lin;                    // [FT][kLinChunk]
  float* inT = sm_lin + FT * kLinChunk;  // [kLinChunk][32]
  const int f0 = blockIdx.x * FT, n0 = blockIdx.y * 32;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  float acc[J];
#pragma unroll
  for (int j = 0; j < J; ++j) acc[j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += kLinChunk) {
    const int kc = min(kLinChunk, K - k0), kc4 = kc >> 2;
    __syncthreads();
    for (int i = tid; i < FT * kc4; i += 256) {
      const int r = i / kc4, c4 = i - r * kc4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (f0 + r < F) v = __ldg(reinterpret_cast<const float4*>(W + (size_t)(f0 + r) * K + k0) + c4);
      reinterpret_cast<float4*>(Ws + r * kLinChunk)[c4] = v;
    }
    for (int i = tid; i < 32 * kc; i += 256) {
      const int nn = i / kc, k = i - nn * kc;
      float v = 0.f;
      if (n0 + nn < B) {
        const int kk = k0 + k;
        if (hw_perm > 0) { const int c = kk / hw_perm, pix = kk - c * hw_perm; v = in[(size_t)(n0 + nn) * K + (size_t)pix * (K / hw_perm) + c]; }
        else v = in[(size_t)(n0 + nn) * K + kk];
      }
      inT[k * 32 + nn] = v;
    }
    __syncthreads();
    for (int k4 = 0; k4 < kc4; ++k4) {
      const float x0 = inT[(4 * k4 + 0) * 32 + lane], x1 = inT[(4 * k4 + 1) * 32 + lane];
      const float x2 = inT[(4 * k4 + 2) * 32 + lane], x3 = inT[(4 * k4 + 3) * 32 + lane];
#pragma unroll
      for (int j = 0; j < J; ++j) {
        const float4 w = reinterpret_cast<const float4*>(Ws + (warp * J + j) * kLinChunk)[k4];
        acc[j] = fmaf(w.x, x0, acc[j]); acc[j] = fmaf(w.y, x1, acc[j]);
        acc[j] = fmaf(w.z, x2, acc[j]); acc[j] = fmaf(w.w, x3, acc[j]);
      }
    }
  }
  if (n0 + lane < B) {
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int f = f0 + warp * J + j;
      if (f < F) {
        float v = acc[j] + (bias ? bias[f] : 0.f);
        float* o = out + (size_t)(n0 + lane) * F + f;
        if (accumulate) v += *o;
        if (silu) v = v / (1.0f + expf(-v));
        *o = v;
      }
    }
  }
}

// MaxPool2d(2) (actor_critic.py:109) on NHWC + GroupNorm partial sums of the pooled tensor (input of the next
// SmallResBlock's GroupNorm).  grid (ceil(Ho*Wo*C/256), B)
__global__ void maxpool2_stats_kernel(const float* __restrict__ x, float* __restrict__ y, double* __restrict__ stats,
                                      int H, int W, int C, int gs) {
  const int n = blockIdx.y;
  const int Ho = H >> 1, Wo = W >> 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int total = Ho * Wo * C;
  float v = 0.f;
  int c = 0;
  const bool ok = i < total;
  if (ok) {
    c = i % C;
    const int pix = i / C, xo = pix % Wo, yo = pix / Wo;
    const float* p = x + (((size_t)n * H + 2 * yo) * W + 2 * xo) * C + c;
    v = fmaxf(fmaxf(p[0], p[C]), fmaxf(p[(size_t)W * C], p[(size_t)W * C + C]));
    y[(size_t)n * total + i] = v;
  }
  if (stats != nullptr) {
    // lanes of a warp hold consecutive channels; gs is a multiple of 32 or divides 32 -> reduce within aligned segments
    const int G = C / gs;
    float s = ok ? v : 0.f, ss = ok ? v * v : 0.f;
    const int seg = gs < 32 ? gs : 32;  // C % seg == 0 and warps start at multiples of 32 channels-wise (256 % C == 0 or C % 32 == 0)
    for (int off = seg >> 1; off > 0; off >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, off);
      ss += __shfl_xor_sync(0xffffffffu, ss, off);
    }
    if (ok && (threadIdx.x & (seg - 1)) == 0) {
      atomicAdd(stats + ((size_t)n * G + c / gs) * 2, (double)s);
      atomicAdd(stats + ((size_t)n * G + c / gs) * 2 + 1, (double)ss);
    }
  }
}

// LSTMCell pointwise part (torch gate order i, f, g, o; actor_critic.py:72): gates [B][4H] already hold
// x W_ih^T + b_ih + h W_hh^T + b_hh.
__global__ void lstm_gates_kernel(const float* __restrict__ gates, const float* __restrict__ c_in, float* __restrict__ h_out,
                                  float* __restrict__ c_out, int B, int Hd) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * Hd) return;
  const int n = i / Hd, j = i - n * Hd;
  const float* g = gates + (size_t)n * 4 * Hd;
  const float ig = 1.f / (1.f + expf(-g[j])), fg = 1.f / (1.f + expf(-g[Hd + j]));
  const float gg = tanhf(g[2 * Hd + j]), og = 1.f / (1.f + expf(-g[3 * Hd + j]));
  const float c = fg * c_in[i] + ig * gg;
  c_out[i] = c;
  h_out[i] = og * tanhf(c);
}

// ------------------------------------------------------------------------------------------------
// SelfAttention2d (blocks.py:51-72), C in {32, 64}, head_dim 8.
//   xn = GroupNorm(x) ; qkv = 1x1 ; att = softmax(q k^T / sqrt(d)) ; y = att v ; out = xn + out_proj(y)
// NOTE the residual is added to the NORMED x (blocks.py:64 rebinding, :72).  Input stats come from the producer's
// epilogue; output stats (for the next AdaGroupNorm) are accumulated here.
struct AttnParams {
  const float* x;       // NHWC [B][L][C]
  const double* st_in;  // [B][G][2]
  const float* gamma;   // [C]
  const float* beta;
  const float* wqkv;    // [3C][C]
  const float* bqkv;    // [3C]
  const float* wout;    // [C][C]
  const float* bout;    // [C]
  float* out;           // NHWC [B][L][C]
  double* ostats;       // [B][G][2] or null
  int L, C, gs;
  float eps;
  long long* ktrace = nullptr;
  float* scratch = nullptr;  // L != 64: q | k | v of every token, [B][3][C/8][L][8] (attn_qkv_kernel -> attn_stream_kernel)
};

constexpr int kAttnThreads = 512;   // attn_bwd_kernel: one CTA per image
constexpr int kAttnL = 64;

// ------------------------------------------------------------------------------------------------
// SelfAttention2d at L = 64 (the 8x8 level of a 64x64 frame) on a CLUSTER of four CTAs per image.
// One CTA per image would keep only 32 SMs busy at the benchmark batch.  Here cluster rank r owns C/4 channels = C/32 heads:
//   every CTA   : GroupNorm(x) for all channels (its q/k/v rows contract over all of them)
//   rank r      : q, k, v rows of its heads -> softmax(q k^T / sqrt(d)) v with the 64 keys split over 2 (C=64) or 4 (C=32)
//                 threads per (head, query) and merged with shuffles -> its C/4 channels of y in ITS shared memory
//   cluster.sync, then every CTA reads the other three y slices through distributed shared memory and computes ITS C/4
//   output channels of out_proj(y) + xn (blocks.py:72: the residual is the NORMED x), plus their GroupNorm partial sums.
// 256 threads per CTA, 4 * B CTAs.
constexpr int kAttnCThreads = 256;

template <int C>
__global__ void __cluster_dims__(4, 1, 1) __launch_bounds__(kAttnCThreads) attn_cluster_kernel(const AttnParams p) {
  namespace cg = cooperative_groups;
  constexpr int L = kAttnL, XP = C + 1, CH = C / 4, HL = CH / 8;      // CH channels / HL heads per CTA
  constexpr int Q3 = 3 * CH, QP = Q3 + 4;                            // local q | k | v row, float4-addressable
  constexpr int KS = kAttnCThreads / (HL * L);                       // threads per (head, query): 1 (C=128), 2 (C=64) or 4 (C=32)
  constexpr int KPT = L / KS;                                        // keys per thread
  extern __shared__ __align__(16) float sm_attn[];
  float* xs = sm_attn;              // [L][XP]  normed x
  float* qkv = xs + L * XP;         // [L][QP]  local q, k, v
  float* ys = qkv + L * QP;         // [L][CH]  local y (read by the other ranks)
  float* ya = ys + L * CH;          // [L][XP]  all channels of y
  float* wq = ya + L * XP;          // [Q3][C]  this rank's rows of the in-projection (staged once, coalesced: the per-thread
  float* wo = wq + Q3 * C;          // [CH][C]  ... and of the out-projection     broadcast reads then come from shared memory)
  __shared__ float smr[8][2];
  cg::cluster_group cluster = cg::this_cluster();
  const int r = (int)cluster.block_rank();
  const int n = blockIdx.x >> 2, tid = threadIdx.x;
  if (blockIdx.x == 0 && tid == 0) ktrace_stamp(p.ktrace);
  // weights first: they do not depend on the previous kernel's output, and every later read is a shared-memory broadcast instead
  // of an L2 round trip per (thread, row, 4 input channels)
  for (int i = tid; i < Q3 * (C / 4); i += kAttnCThreads) {
    const int j = i / (C / 4), c4 = i - j * (C / 4);
    const int part = j / CH, cc = j - part * CH;
    reinterpret_cast<float4*>(wq)[i] = __ldg(reinterpret_cast<const float4*>(p.wqkv + (size_t)(part * C + r * CH + cc) * C) + c4);
  }
  for (int i = tid; i < CH * (C / 4); i += kAttnCThreads) {
    const int j = i / (C / 4), c4 = i - j * (C / 4);
    reinterpret_cast<float4*>(wo)[i] = __ldg(reinterpret_cast<const float4*>(p.wout + (size_t)(r * CH + j) * C) + c4);
  }
  const int G = C / p.gs;
  if (tid < G) {
    const double cnt = (double)L * p.gs;
    const double mean = p.st_in[((size_t)n * G + tid) * 2] / cnt;
    double var = p.st_in[((size_t)n * G + tid) * 2 + 1] / cnt - mean * mean;
    var = var > 0.0 ? var : 0.0;
    smr[tid][0] = (float)mean;
    smr[tid][1] = (float)(1.0 / sqrt(var + (double)p.eps));
  }
  __syncthreads();
  const float* xg = p.x + (size_t)n * L * C;
  for (int i = tid; i < L * C; i += kAttnCThreads) {
    const int l = i / C, c = i - l * C;
    const int g = c / p.gs;
    xs[l * XP + c] = (xg[i] - smr[g][0]) * smr[g][1] * __ldg(p.gamma + c) + __ldg(p.beta + c);
  }
  __syncthreads();
  // ---- local q | k | v rows: thread = (token l, output group og of NO outputs)
  {
    constexpr int NG = kAttnCThreads / L;   // 4
    constexpr int NO = Q3 / NG;             // 24 (C=128), 12 (C=64) or 6 (C=32)
    const int l = tid % L, og = tid / L;
    float acc[NO];
    int row[NO];
#pragma unroll
    for (int i = 0; i < NO; ++i) {
      const int j = og * NO + i, part = j / CH, cc = j - part * CH;
      row[i] = part * C + r * CH + cc;      // row of the [3C][C] in-projection (q rows, then k rows, then v rows)
      acc[i] = __ldg(p.bqkv + row[i]);
    }
    for (int c4 = 0; c4 < C / 4; ++c4) {
      const float x0 = xs[l * XP + 4 * c4], x1 = xs[l * XP + 4 * c4 + 1], x2 = xs[l * XP + 4 * c4 + 2], x3 = xs[l * XP + 4 * c4 + 3];
#pragma unroll
      for (int i = 0; i < NO; ++i) {
        const float4 w = reinterpret_cast<const float4*>(wq + (og * NO + i) * C)[c4];
        acc[i] = fmaf(w.x, x0, acc[i]); acc[i] = fmaf(w.y, x1, acc[i]);
        acc[i] = fmaf(w.z, x2, acc[i]); acc[i] = fmaf(w.w, x3, acc[i]);
      }
    }
#pragma unroll
    for (int i = 0; i < NO; ++i) qkv[l * QP + og * NO + i] = acc[i];
  }
  __syncthreads();
  // ---- attention: item = (local head hl, query l), KS neighbouring lanes split the keys and merge (max, sum, y) by shuffles
  {
    const int item = tid / KS, part = tid % KS;
    const int hl = item / L, l = item - hl * L;
    float q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) q[e] = qkv[l * QP + hl * 8 + e] * 0.35355339059327373f;  // 1/sqrt(8)
    float sc[KPT];
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < KPT; ++jj) {
      const int j = part * KPT + jj;
      const float4 k0 = *reinterpret_cast<const float4*>(qkv + j * QP + CH + hl * 8);
      const float4 k1 = *reinterpret_cast<const float4*>(qkv + j * QP + CH + hl * 8 + 4);
      float sj = q[0] * k0.x;
      sj = fmaf(q[1], k0.y, sj); sj = fmaf(q[2], k0.z, sj); sj = fmaf(q[3], k0.w, sj);
      sj = fmaf(q[4], k1.x, sj); sj = fmaf(q[5], k1.y, sj); sj = fmaf(q[6], k1.z, sj); sj = fmaf(q[7], k1.w, sj);
      sc[jj] = sj;
      mx = fmaxf(mx, sj);
    }
#pragma unroll
    for (int m = 1; m < KS; m <<= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, m));   // the row maximum over all 64 keys
    float den = 0.f;
    float y[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int jj = 0; jj < KPT; ++jj) {
      const int j = part * KPT + jj;
      const float pj = expf(sc[jj] - mx);
      den += pj;
      const float4 v0 = *reinterpret_cast<const float4*>(qkv + j * QP + 2 * CH + hl * 8);
      const float4 v1 = *reinterpret_cast<const float4*>(qkv + j * QP + 2 * CH + hl * 8 + 4);
      y[0] = fmaf(pj, v0.x, y[0]); y[1] = fmaf(pj, v0.y, y[1]); y[2] = fmaf(pj, v0.z, y[2]); y[3] = fmaf(pj, v0.w, y[3]);
      y[4] = fmaf(pj, v1.x, y[4]); y[5] = fmaf(pj, v1.y, y[5]); y[6] = fmaf(pj, v1.z, y[6]); y[7] = fmaf(pj, v1.w, y[7]);
    }
#pragma unroll
    for (int m = 1; m < KS; m <<= 1) {
      den += __shfl_xor_sync(0xffffffffu, den, m);
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] += __shfl_xor_sync(0xffffffffu, y[e], m);
    }
    if (part == 0) {
      const float inv = 1.0f / den;
#pragma unroll
      for (int e = 0; e < 8; ++e) ys[l * CH + hl * 8 + e] = y[e] * inv;
    }
  }
  cluster.sync();   // every rank's y slice is complete and visible cluster-wide
  // ---- gather all channels of y (three slices through distributed shared memory)
  for (int i = tid; i < L * C; i += kAttnCThreads) {
    const int l = i / C, c = i - l * C;
    const int src = c / CH;
    const float* remote = cluster.map_shared_rank(ys, src);
    ya[l * XP + c] = remote[l * CH + (c - src * CH)];
  }
  cluster.sync();   // nobody leaves (or overwrites ys) while its slice is still being read
  // ---- out projection of THIS rank's channels + residual on normed x; statistics.  thread = (token l, NO2 outputs)
  {
    constexpr int NG = kAttnCThreads / L;   // 4
    constexpr int NO2 = CH / NG;            // 8 (C=128), 4 (C=64) or 2 (C=32) consecutive outputs
    const int l = tid % L, og = tid / L;
    const int oc0 = r * CH + og * NO2;
    float acc[NO2];
#pragma unroll
    for (int i = 0; i < NO2; ++i) acc[i] = __ldg(p.bout + oc0 + i);
    for (int c4 = 0; c4 < C / 4; ++c4) {
      const float y0 = ya[l * XP + 4 * c4], y1 = ya[l * XP + 4 * c4 + 1], y2 = ya[l * XP + 4 * c4 + 2], y3 = ya[l * XP + 4 * c4 + 3];
#pragma unroll
      for (int i = 0; i < NO2; ++i) {
        const float4 w = reinterpret_cast<const float4*>(wo + (og * NO2 + i) * C)[c4];
        acc[i] = fmaf(w.x, y0, acc[i]); acc[i] = fmaf(w.y, y1, acc[i]);
        acc[i] = fmaf(w.z, y2, acc[i]); acc[i] = fmaf(w.w, y3, acc[i]);
      }
    }
    float* og_ptr = p.out + (size_t)n * L * C + (size_t)l * C + oc0;
    float a = 0.f, b = 0.f;
#pragma unroll
    for (int i = 0; i < NO2; ++i) {
      const float v = xs[l * XP + oc0 + i] + acc[i];
      og_ptr[i] = v;
      a += v; b += v * v;
    }
    if (p.ostats) {   // all channels of a CTA lie in one GroupNorm group (CH <= gs, gs a multiple of CH)
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, off);
        b += __shfl_xor_sync(0xffffffffu, b, off);
      }
      if ((tid & 31) == 0) {
        const int g = (r * CH) / p.gs;
        atomicAdd(p.ostats + ((size_t)n * G + g) * 2, (double)a);
        atomicAdd(p.ostats + ((size_t)n * G + g) * 2 + 1, (double)b);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// SelfAttention2d over any token count L >= 1 (same math as attn_cluster_kernel, same parameter block plus p.scratch), in two launches
// of grid (ceil(L / 32), B):
//   attn_qkv_kernel   : 32 tokens per CTA: GroupNorm(x) from the producer's statistics, the qkv 1x1 projection into p.scratch,
//                       head-major [B][3][C/8][L][8] (q, k, v), so that the keys of one head are contiguous
//   attn_stream_kernel: 32 queries per CTA, all heads: K / V tiles of every head streamed through shared memory, the running
//                       max, sum and y of each (head, query) in registers (keys past L masked), split over KS neighbouring
//                       threads that share the running max and merge their sums with shuffles at the end; then
//                       out_proj(y) + xn (xn recomputed from x and the statistics) and the output's GroupNorm partial sums.
// 32 queries per CTA: at the 19x35 = 665 tokens of a 150x280 frame, 8 images give 168 CTAs for the 132 SMs.
constexpr int kAttnTile = 32;        // tokens (queries) per CTA
constexpr int kAttnQkvThreads = 256;
constexpr int kAttnSThreads = 512;

// (float) mean and rstd of every group of image n (as attn_cluster_kernel computes them), for the first C / gs threads
__device__ __forceinline__ void attn_group_stats(const AttnParams& p, int n, float (*smr)[2]) {
  const int G = p.C / p.gs;
  if ((int)threadIdx.x < G) {
    const double cnt = (double)p.L * p.gs;
    const double mean = p.st_in[((size_t)n * G + threadIdx.x) * 2] / cnt;
    double var = p.st_in[((size_t)n * G + threadIdx.x) * 2 + 1] / cnt - mean * mean;
    var = var > 0.0 ? var : 0.0;
    smr[threadIdx.x][0] = (float)mean;
    smr[threadIdx.x][1] = (float)(1.0 / sqrt(var + (double)p.eps));
  }
}

template <int C>
__global__ void __launch_bounds__(kAttnQkvThreads) attn_qkv_kernel(const AttnParams p) {
  constexpr int TQ = kAttnTile, C3 = 3 * C, XP = C + 1, HEADS = C / 8;
  constexpr int NG = kAttnQkvThreads / TQ;   // 8 output groups
  constexpr int NO = C3 / NG;                // 48 (C=128), 24 (C=64) or 12 (C=32) outputs per thread
  __shared__ float xs[TQ * XP];
  __shared__ float smr[8][2];
  const int n = blockIdx.y, l0 = blockIdx.x * TQ, tid = threadIdx.x, L = p.L;
  if (n == 0 && blockIdx.x == 0 && tid == 0) ktrace_stamp(p.ktrace);
  attn_group_stats(p, n, smr);
  __syncthreads();
  const float* xg = p.x + (size_t)n * L * C;
  for (int i = tid; i < TQ * C; i += kAttnQkvThreads) {
    const int l = i / C, c = i - l * C;
    const int g = c / p.gs;
    xs[l * XP + c] = l0 + l < L ? (xg[(size_t)(l0 + l) * C + c] - smr[g][0]) * smr[g][1] * __ldg(p.gamma + c) + __ldg(p.beta + c) : 0.f;
  }
  __syncthreads();
  // thread = (token l, output group og of NO outputs); a warp = 32 tokens of one og (weights broadcast)
  const int l = tid % TQ, og = tid / TQ;
  float acc[NO];
#pragma unroll
  for (int i = 0; i < NO; ++i) acc[i] = __ldg(p.bqkv + og * NO + i);
  for (int c4 = 0; c4 < C / 4; ++c4) {
    const float x0 = xs[l * XP + 4 * c4], x1 = xs[l * XP + 4 * c4 + 1], x2 = xs[l * XP + 4 * c4 + 2], x3 = xs[l * XP + 4 * c4 + 3];
#pragma unroll
    for (int i = 0; i < NO; ++i) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(p.wqkv + (size_t)(og * NO + i) * C) + c4);
      acc[i] = fmaf(w.x, x0, acc[i]); acc[i] = fmaf(w.y, x1, acc[i]);
      acc[i] = fmaf(w.z, x2, acc[i]); acc[i] = fmaf(w.w, x3, acc[i]);
    }
  }
  if (l0 + l >= L) return;
  float* dst = p.scratch + (size_t)n * C3 * L;
#pragma unroll
  for (int i = 0; i < NO; ++i) {
    const int o = og * NO + i, part = o / C, c = o - part * C;   // row of the [3C][C] in-projection: q rows, then k, then v
    dst[((size_t)(part * HEADS + (c >> 3)) * L + l0 + l) * 8 + (c & 7)] = acc[i];
  }
}

template <int C>
__global__ void __launch_bounds__(kAttnSThreads) attn_stream_kernel(const AttnParams p) {
  constexpr int TQ = kAttnTile, XP = C + 1, HEADS = C / 8;
  constexpr int KS = kAttnSThreads / (HEADS * TQ);   // threads per (head, query): 1 (C=128), 2 (C=64) or 4 (C=32)
  constexpr int KPT = C == 128 ? 16 : 32, TK = KS * KPT;   // keys per thread / tile: 32 KB of K / V, 16 KB at C=128 (48 KB static)
  __shared__ __align__(16) float kv[2 * HEADS * TK * 8];   // [k | v][head][TK][8]
  __shared__ float ys[TQ * XP];
  __shared__ float smr[8][2];
  const int n = blockIdx.y, l0 = blockIdx.x * TQ, tid = threadIdx.x, L = p.L;
  if (n == 0 && blockIdx.x == 0 && tid == 0) ktrace_stamp(p.ktrace);
  attn_group_stats(p, n, smr);
  const float* qkv = p.scratch + (size_t)n * 3 * C * L;
  const int part = tid % KS, item = tid / KS;
  const int h = item / TQ, ql = item - h * TQ;
  float q[8];
  {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    if (l0 + ql < L) {
      const float4* src = reinterpret_cast<const float4*>(qkv + ((size_t)h * L + l0 + ql) * 8);
      a = __ldg(src); b = __ldg(src + 1);
    }
    q[0] = a.x; q[1] = a.y; q[2] = a.z; q[3] = a.w; q[4] = b.x; q[5] = b.y; q[6] = b.z; q[7] = b.w;
#pragma unroll
    for (int e = 0; e < 8; ++e) q[e] *= 0.35355339059327373f;  // 1/sqrt(8)
  }
  float m = -INFINITY, den = 0.f;
  float y[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int j0 = 0; j0 < L; j0 += TK) {
    __syncthreads();   // the previous tile has been consumed
    for (int i = tid; i < 2 * HEADS * TK * 2; i += kAttnSThreads) {   // float4 units, two per key row; zeros past L
      const int f4 = i & 1, r = i >> 1;
      const int j = r % TK, hh = r / TK;                              // hh = k|v part * HEADS + head
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (j0 + j < L) v = __ldg(reinterpret_cast<const float4*>(qkv + ((size_t)(HEADS + hh) * L + j0 + j) * 8) + f4);
      reinterpret_cast<float4*>(kv)[i] = v;
    }
    __syncthreads();
    const float* ks = kv + h * TK * 8;
    const float* vs = kv + (HEADS + h) * TK * 8;
    float sc[KPT];
    float mt = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < KPT; ++jj) {
      const int j = jj * KS + part;
      const float4 k0 = *reinterpret_cast<const float4*>(ks + j * 8);
      const float4 k1 = *reinterpret_cast<const float4*>(ks + j * 8 + 4);
      float sj = q[0] * k0.x;
      sj = fmaf(q[1], k0.y, sj); sj = fmaf(q[2], k0.z, sj); sj = fmaf(q[3], k0.w, sj);
      sj = fmaf(q[4], k1.x, sj); sj = fmaf(q[5], k1.y, sj); sj = fmaf(q[6], k1.z, sj); sj = fmaf(q[7], k1.w, sj);
      sc[jj] = j0 + j < L ? sj : -INFINITY;
      mt = fmaxf(mt, sc[jj]);
    }
#pragma unroll
    for (int s = 1; s < KS; s <<= 1) mt = fmaxf(mt, __shfl_xor_sync(0xffffffffu, mt, s));
    // every tile holds key j0 < L, so the new maximum is finite; on the first tile m = -inf and the correction is 0
    const float mn = fmaxf(m, mt);
    const float corr = expf(m - mn);
    m = mn;
    den *= corr;
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] *= corr;
#pragma unroll
    for (int jj = 0; jj < KPT; ++jj) {
      const int j = jj * KS + part;
      const float pj = expf(sc[jj] - m);
      den += pj;
      const float4 v0 = *reinterpret_cast<const float4*>(vs + j * 8);
      const float4 v1 = *reinterpret_cast<const float4*>(vs + j * 8 + 4);
      y[0] = fmaf(pj, v0.x, y[0]); y[1] = fmaf(pj, v0.y, y[1]); y[2] = fmaf(pj, v0.z, y[2]); y[3] = fmaf(pj, v0.w, y[3]);
      y[4] = fmaf(pj, v1.x, y[4]); y[5] = fmaf(pj, v1.y, y[5]); y[6] = fmaf(pj, v1.z, y[6]); y[7] = fmaf(pj, v1.w, y[7]);
    }
  }
#pragma unroll
  for (int s = 1; s < KS; s <<= 1) {
    den += __shfl_xor_sync(0xffffffffu, den, s);
#pragma unroll
    for (int e = 0; e < 8; ++e) y[e] += __shfl_xor_sync(0xffffffffu, y[e], s);
  }
  if (part == 0) {
    const float inv = 1.0f / den;
#pragma unroll
    for (int e = 0; e < 8; ++e) ys[ql * XP + h * 8 + e] = y[e] * inv;
  }
  __syncthreads();
  // ---- out projection + residual on normed x; statistics.  thread = (token l, NO2 outputs); a warp = 32 tokens of one og
  constexpr int NG = kAttnSThreads / TQ;   // 16
  constexpr int NO2 = C / NG;              // 8, 4 or 2 consecutive outputs: inside one GroupNorm group (gs % 8 == 0)
  const int l = tid % TQ, og = tid / TQ;
  float acc[NO2];
#pragma unroll
  for (int i = 0; i < NO2; ++i) acc[i] = __ldg(p.bout + og * NO2 + i);
  for (int c4 = 0; c4 < C / 4; ++c4) {
    const float y0 = ys[l * XP + 4 * c4], y1 = ys[l * XP + 4 * c4 + 1], y2 = ys[l * XP + 4 * c4 + 2], y3 = ys[l * XP + 4 * c4 + 3];
#pragma unroll
    for (int i = 0; i < NO2; ++i) {
      const float4 w = __ldg(reinterpret_cast<const float4*>(p.wout + (size_t)(og * NO2 + i) * C) + c4);
      acc[i] = fmaf(w.x, y0, acc[i]); acc[i] = fmaf(w.y, y1, acc[i]);
      acc[i] = fmaf(w.z, y2, acc[i]); acc[i] = fmaf(w.w, y3, acc[i]);
    }
  }
  float a = 0.f, b = 0.f;
  if (l0 + l < L) {
    const size_t row = ((size_t)n * L + l0 + l) * C + og * NO2;
#pragma unroll
    for (int i = 0; i < NO2; ++i) {
      const int c = og * NO2 + i, g = c / p.gs;
      const float xn = (p.x[row + i] - smr[g][0]) * smr[g][1] * __ldg(p.gamma + c) + __ldg(p.beta + c);
      const float v = xn + acc[i];
      p.out[row + i] = v;
      a += v; b += v * v;
    }
  }
  if (p.ostats) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, off);
      b += __shfl_xor_sync(0xffffffffu, b, off);
    }
    if ((tid & 31) == 0) {
      const int G = C / p.gs, g = (og * NO2) / p.gs;
      atomicAdd(p.ostats + ((size_t)n * G + g) * 2, (double)a);
      atomicAdd(p.ostats + ((size_t)n * G + g) * 2 + 1, (double)b);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// wrap_model_output (denoiser.py:79-84) + one sampler update (diffusion_sampler.py:45-49 Euler, :50-56 Heun pieces).
//   F: NHWC [B][HW][CF] model output (first Cimg channels used)  x: NCHW noisy input
//   denoised = quantise(clamp(c_skip*x + c_out*F))      (always written if non-null)
//   mode 0: nothing else
//   mode 1: Euler          x_out = x + ((x - denoised)/sigma_hat) * dt                      (d_out = d if non-null)
//   mode 2: Heun 2nd stage x_out = x0 + ((d_prev + (x - denoised)/sigma_hat)/2) * dt        (x = x_2, x0 = stage input)
__global__ void wrap_update_kernel(const float* __restrict__ F, const float* __restrict__ x, const float* __restrict__ cs,
                                   float* __restrict__ model_out_nchw, float* __restrict__ denoised,
                                   float* __restrict__ x_out, float* __restrict__ d_out, const float* __restrict__ d_prev,
                                   const float* __restrict__ x0, int mode, float sigma_hat, float dt, int Cimg, int CF,
                                   int HW, int total, long long* ktrace) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // NCHW linear index
  if (i == 0) ktrace_stamp(ktrace);
  if (i >= total) return;
  const int pix = i % HW, c = (i / HW) % Cimg, n = i / (HW * Cimg);
  const float f = F[((size_t)n * HW + pix) * CF + c];
  if (model_out_nchw) model_out_nchw[i] = f;
  const float c_out = cs[n * 4 + 1], c_skip = cs[n * 4 + 2];
  const float xv = x[i];
  float d = __fadd_rn(__fmul_rn(c_skip, xv), __fmul_rn(c_out, f));
  d = fminf(fmaxf(d, -1.0f), 1.0f);
  float t = __fmul_rn(__fdiv_rn(__fadd_rn(d, 1.0f), 2.0f), 255.0f);
  const float qv = (float)(unsigned char)t;  // .byte(): truncation
  const float den = __fsub_rn(__fmul_rn(__fdiv_rn(qv, 255.0f), 2.0f), 1.0f);
  if (denoised) denoised[i] = den;
  if (mode == 0) return;
  const float dd = __fdiv_rn(__fsub_rn(xv, den), sigma_hat);
  if (mode == 1) {
    if (d_out) d_out[i] = dd;
    x_out[i] = __fadd_rn(xv, __fmul_rn(dd, dt));
  } else {
    const float dp = __fdiv_rn(__fadd_rn(d_prev[i], dd), 2.0f);
    x_out[i] = __fadd_rn(x0[i], __fmul_rn(dp, dt));
  }
}

// x_out = x + eps * s   (sampler churn, diffusion_sampler.py:41-43)
__global__ void axpy_kernel(const float* __restrict__ x, const float* __restrict__ e, float s, float* __restrict__ o,
                            int total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < total) o[i] = __fadd_rn(x[i], __fmul_rn(e[i], s));
}

// ------------------------------------------------------------------------------------------------
// Weight packing: torch Conv2d weight [Cout][CinReal][kh][kw] fp32 -> UMMA B operand [tap][Cin/8][CoutPad][8] fp16.
// Input channel ci of the packed tensor maps to real channel ci if ci < c0_real, zero if c0_real <= ci < c0_store,
// and c0_real + (ci - c0_store) for the second source (concat), zero beyond.
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, __half* __restrict__ wpk, int Cout, int CoutPad,
                                        int CinReal, int Cin, int taps, int c0_real, int c0_store, int precise) {
  // precise: K = 3*Cin laid out as [W_hi | W_hi | W_lo] to meet operands [A_hi | A_lo | A_hi] (split-fp16 product
  // A W ~= A_hi W_hi + A_lo W_hi + A_hi W_lo, error ~2^-22 instead of 2^-11)
  // precise == 2: the LOW parts alone, K = Cin (third pass of a three-launch split-fp16 conv whose 3*Cin weights would not fit
  // in shared memory)
  const int K = precise == 1 ? 3 * Cin : Cin;
  const int total = taps * K * CoutPad;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int e = i & 7;
    const int co = (i >> 3) % CoutPad;
    const int j = (i >> 3) / CoutPad % (K >> 3);
    const int t = (i >> 3) / CoutPad / (K >> 3);
    const int kk = j * 8 + e;
    const int seg = kk / Cin, ci = kk - seg * Cin;
    int cr = -1;
    if (ci < c0_store) cr = ci < c0_real ? ci : -1;
    else cr = c0_real + (ci - c0_store);
    float v = 0.f;
    if (co < Cout && cr >= 0 && cr < CinReal) v = w[((size_t)co * CinReal + cr) * taps + t];
    const __half hi = __float2half_rn(v);
    wpk[i] = (precise != 2 && seg < 2) ? hi : __float2half_rn(v - __half2float(hi));
  }
}

// GroupNorm partial sums of an NHWC tensor (used for tensors that do not come out of a conv epilogue, and by tests).
// stats[n][g] += (sum, sumsq).  grid: (chunks, B)
__global__ void gn_stats_kernel(const float* __restrict__ x, double* __restrict__ stats, int HW, int C, int gs) {
  const int n = blockIdx.y;
  const int G = C / gs;
  const size_t per = (size_t)HW * C;
  const float* xb = x + (size_t)n * per;
  // each thread walks elements with a fixed channel when C divides the stride; generic otherwise
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (int g = 0; g < G; ++g) {
    float s = 0.f, ss = 0.f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < per; i += stride) {
      const int c = (int)(i % C);
      if (c / gs == g) { const float v = xb[i]; s += v; ss += v * v; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, off);
      ss += __shfl_xor_sync(0xffffffffu, ss, off);
    }
    if ((threadIdx.x & 31) == 0) {
      atomicAdd(stats + ((size_t)n * G + g) * 2, (double)s);
      atomicAdd(stats + ((size_t)n * G + g) * 2 + 1, (double)ss);
    }
  }
}

// Deterministic GroupNorm sums (torch.use_deterministic_algorithms).  Each (group, image) is owned by one cluster of
// kGnDetSplit CTAs; CTA r of the cluster takes the r-th of kGnDetSplit fixed, contiguous pixel ranges.  Thread t sums elements
// t, t + blockDim, ... of its range in fp32 (four consecutive channels per load: C and gs are multiples of 4), the CTA adds
// its threads' sums in a fixed fp64 tree, and rank 0 adds the CTAs' sums in rank order through distributed shared memory.  So
// the result depends on the tensor alone, not on scheduling or the SM count, and no partials buffer is needed.
// stats[n][g] += (sum, sumsq) with a plain add (rank 0 is the slot's only writer).  grid: (kGnDetSplit * C / gs, B).
// Not a template: an instantiation placed ahead of linear_kernel's in the translation unit changed that kernel's SASS.
constexpr int kGnDetThreads = 256, kGnDetSplit = 8;
__global__ void __cluster_dims__(kGnDetSplit, 1, 1) __launch_bounds__(kGnDetThreads)
gn_stats_det_kernel(const float* __restrict__ x, double* __restrict__ stats, int HW, int C, int gs) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  const int r = (int)cluster.block_rank();
  const int g = blockIdx.x / kGnDetSplit, n = blockIdx.y, G = C / gs;
  const int q = gs >> 2;
  const int per = (HW + kGnDetSplit - 1) / kGnDetSplit, p0 = min(HW, r * per), p1 = min(HW, p0 + per);
  const float* xb = x + ((size_t)n * HW + p0) * C + (size_t)g * gs;
  const long long total = (long long)(p1 - p0) * q;
  float s = 0.f, ss = 0.f;
#pragma unroll 4
  for (long long i = threadIdx.x; i < total; i += kGnDetThreads) {
    const long long pix = i / q;
    const float4 v = __ldg(reinterpret_cast<const float4*>(xb + pix * C) + (i - pix * q));
    s += (v.x + v.y) + (v.z + v.w);
    ss += fmaf(v.x, v.x, v.y * v.y) + fmaf(v.z, v.z, v.w * v.w);
  }
  __shared__ double rs[kGnDetThreads], rss[kGnDetThreads];
  rs[threadIdx.x] = s; rss[threadIdx.x] = ss;
  __syncthreads();
  for (int m = kGnDetThreads / 2; m > 0; m >>= 1) {
    if ((int)threadIdx.x < m) { rs[threadIdx.x] += rs[threadIdx.x + m]; rss[threadIdx.x] += rss[threadIdx.x + m]; }
    __syncthreads();
  }
  cluster.sync();   // every CTA's sums are complete and visible cluster-wide
  if (r == 0 && threadIdx.x == 0) {
    double a = 0.0, b = 0.0;
    for (int k = 0; k < kGnDetSplit; ++k) { a += *cluster.map_shared_rank(rs, k); b += *cluster.map_shared_rank(rss, k); }
    double* dst = stats + ((size_t)n * G + g) * 2;
    dst[0] += a;
    dst[1] += b;
  }
  cluster.sync();   // no CTA leaves while rank 0 still reads its shared memory
}

}  // namespace dmd
