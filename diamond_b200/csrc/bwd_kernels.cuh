// CUDA-core kernels of the backward pass (everything that is not a conv dgrad / wgrad): GroupNorm / AdaGroupNorm + SiLU
// backward as two passes, column sums (bias gradients), the upsample adjoint, a small strided SGEMM for the linear
// layers, embedding / LSTM / max-pool / attention backward.  Each kernel cites the reference forward lines whose
// autograd it reproduces.  All gradient tensors are fp32 and carry the loss scale S (a device scalar: scale[0] = S,
// scale[1] = 1/S) chosen from the incoming gradient so that their fp16 tensor-core operands stay in range; parameter
// gradients are multiplied by 1/S where they are written.
#pragma once
#include "../../include/diamond_b200.h"
#include "aux_kernels.cuh"

namespace dmd {

// ------------------------------------------------------------------------------------------------ loss scale
// amax of |g| (non-negative floats order like their bit patterns) -> S = 2^(E - e) with amax = f * 2^e, f in [0.5, 1) and
// E = DMD_LOSS_SCALE_EXP, so max |S g| = f * 2^E lies in [2^(E-1), 2^E).  A power of two amax = 2^k gets f = 0.5, e = k + 1.
__global__ void absmax_kernel(const float* __restrict__ g, unsigned int* __restrict__ amax_bits, long long n) {
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) m = fmaxf(m, fabsf(g[i]));
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0 && m > 0.f && m < INFINITY) atomicMax(amax_bits, __float_as_uint(m));
}
__global__ void loss_scale_kernel(const unsigned int* __restrict__ amax_bits, float* __restrict__ scale) {
  const float m = __uint_as_float(*amax_bits);
  float s = 1.f;
  if (m > 0.f) {
    int e;
    frexpf(m, &e);                 // m = f * 2^e, f in [0.5, 1)
    s = ldexpf(1.f, DMD_LOSS_SCALE_EXP - e);
  }
  scale[0] = s;
  scale[1] = 1.f / s;
}
// NCHW (B, C, HW) -> NHWC with CP channels (zero padded), multiplied by scale[0]: the gradient of the model output
__global__ void nchw_to_nhwc_scaled_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ scale,
                                           int C, int CP, int HW) {
  const int n = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= HW) return;
  const float s = scale[0];
  float* o = out + ((size_t)n * HW + pix) * CP;
  for (int ch = 0; ch < CP; ++ch) o[ch] = ch < C ? in[((size_t)n * C + ch) * HW + pix] * s : 0.f;
}
// NHWC (C channels of CP) -> NCHW, multiplied by scale[1] (gradient wrt an input tensor, unscaled)
__global__ void nhwc_to_nchw_scaled_kernel(const float* __restrict__ in, float* __restrict__ out, const float* __restrict__ scale,
                                           int C, int CP, int HW) {
  const int n = blockIdx.y;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= HW) return;
  const float s = scale ? scale[1] : 1.f;
  const float* i = in + ((size_t)n * HW + pix) * CP;
  for (int ch = 0; ch < C; ++ch) out[((size_t)n * C + ch) * HW + pix] = i[ch] * s;
}

// ------------------------------------------------------------------------------------------------ column sums
// out[c] += alpha * sum_rows x[row][c]   (bias gradients: nn.Conv2d / nn.Linear bias, sum of dL/dy over batch and pixels)
// x: [rows][C] fp32, C multiple of 4.  out2 (optional) receives the same sums.  grid: (row chunks, ceil(C / 256)).
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, float* __restrict__ out, float* __restrict__ out2,
                                                     const float* __restrict__ inv_scale, long long rows, int C, int Creal) {
  __shared__ float cs_sm[1024];      // [row lanes][Cb] partials -> reduced over the row lanes
  const int cbase = blockIdx.y * 256;
  const int Cb = min(256, C - cbase);
  const int L4 = Cb >> 2;
  const int lanes = 256 / L4;        // row lanes per block (1 when Cb = 256 ... 64 when Cb = 16)
  const int c4 = threadIdx.x % L4, rl = threadIdx.x / L4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (rl < lanes) {
    for (long long r = (long long)blockIdx.x * lanes + rl; r < rows; r += (long long)gridDim.x * lanes) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * C + cbase) + c4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    reinterpret_cast<float4*>(cs_sm + (size_t)rl * Cb)[c4] = acc;
  }
  __syncthreads();
  if ((int)threadIdx.x < Cb) {
    float s = 0.f;
    for (int k = 0; k < lanes; ++k) s += cs_sm[(size_t)k * Cb + threadIdx.x];
    const int c = cbase + threadIdx.x;
    if (c < Creal) {
      s *= inv_scale ? *inv_scale : 1.f;
      atomicAdd(out + c, s);
      if (out2) atomicAdd(out2 + c, s);
    }
  }
}

// ------------------------------------------------------------------------------------------------ norm + SiLU backward
// Forward (prep_act_kernel): y = silu(z), z = k[n,c] * xhat + sh[n,c], xhat = (x - mean[n,g]) * rstd[n,g]
//   AdaGroupNorm (blocks.py:41-45): k = 1 + scale, sh = shift, (scale, shift) = FiLM linear output
//   GroupNorm    (blocks.py:28)   : k = gamma[c],  sh = beta[c]
// Backward given gy = dL/dy (oracle/backward_plan.py adagn_silu_backward_two_pass):
//   gz = gy * silu'(z)
//   pass 1:  A[n,c] = sum_px gz   (= d shift / d beta contribution),  Bm[n,c] = sum_px gz * xhat  (= d scale / d gamma)
//   pass 2:  m1[n,g] = sum_{c in g} k A / cnt,  m2[n,g] = sum_{c in g} k Bm / cnt
//            gx = rstd * (k gz - m1 - xhat m2)      [+ addend]   (assign or accumulate)
struct NormBwdParams {
  const float* x;        // NHWC [B][HW][C] forward input of the norm
  const float* gy;       // NHWC [B][HW][C] gradient wrt the activated output
  const double* stats;   // [B][C/gs][2] forward (sum, sumsq)
  int B, HW, C, gs;
  int mode;              // 1 AdaGroupNorm, 2 affine GroupNorm
  int act;               // SiLU applied after the norm
  const float* film;     // [B][film_stride]: scale at film_off + c_off + c, shift at film_off + ctot + c_off + c
  int film_stride, film_off, film_ctot, c_off;
  const float* gamma;    // [C] (mode 2; indexed c_off + c)
  const float* beta;
  float eps;
  float* sumA;           // pass-1 outputs: sumA[n * sum_stride + c], sumB[n * sum_stride + c]  (atomically accumulated)
  float* sumB;
  int sum_stride;
  float* gx;             // pass-2 output NHWC [B][HW][C]
  const float* addend;   // optional NHWC tensor added to gx (identity residual path) or null
  int accumulate;        // gx += instead of gx =
};

__device__ __forceinline__ float dsilu_f(float z) {
  const float s = 1.f / (1.f + __expf(-z));
  return s * (1.f + z * (1.f - s));
}

constexpr int kNormThreads = 256;

// coefficients of image n into shared memory: a = rstd*k, b = sh - mean*a, kk = k, rs = rstd, mu = mean
__device__ __forceinline__ void norm_coeffs(const NormBwdParams& p, int n, float* sa, float* sb, float* sk, float* srs, float* smu) {
  const int G = p.C / p.gs;
  __shared__ float smr[8][2];
  if ((int)threadIdx.x < G) {
    const double* st = p.stats + ((size_t)n * G + threadIdx.x) * 2;
    const double cnt = (double)p.HW * p.gs;
    const double mean = st[0] / cnt;
    double var = st[1] / cnt - mean * mean;
    var = var > 0.0 ? var : 0.0;
    smr[threadIdx.x][0] = (float)mean;
    smr[threadIdx.x][1] = (float)(1.0 / sqrt(var + (double)p.eps));
  }
  __syncthreads();
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    const float mean = smr[c / p.gs][0], rstd = smr[c / p.gs][1];
    float k, sh;
    if (p.mode == 1) {
      const float* f = p.film + (size_t)n * p.film_stride + p.film_off;
      k = 1.f + __ldg(f + p.c_off + c);
      sh = __ldg(f + p.film_ctot + p.c_off + c);
    } else {
      k = __ldg(p.gamma + p.c_off + c);
      sh = __ldg(p.beta + p.c_off + c);
    }
    const float a = rstd * k;
    sa[c] = a; sb[c] = sh - mean * a; sk[c] = k; srs[c] = rstd; smu[c] = mean;
  }
  __syncthreads();
}

// grid (chunks, B); each block walks pixels pix = blockIdx.x*ppb .. of image blockIdx.y; thread = (channel quad, pixel lane)
__global__ void __launch_bounds__(kNormThreads) norm_bwd_pass1_kernel(const NormBwdParams p, int ppb) {
  __shared__ float sa[kMaxCin], sb[kMaxCin], sk[kMaxCin], srs[kMaxCin], smu[kMaxCin];
  __shared__ float red[kNormThreads][8];
  const int n = blockIdx.y;
  norm_coeffs(p, n, sa, sb, sk, srs, smu);
  const int L4 = p.C >> 2, lanes = kNormThreads / L4;
  const int c4 = threadIdx.x % L4, pl = threadIdx.x / L4;
  const int c = c4 * 4;
  float A[4] = {0.f, 0.f, 0.f, 0.f}, Bm[4] = {0.f, 0.f, 0.f, 0.f};
  const int p0 = blockIdx.x * ppb, p1 = min(p0 + ppb, p.HW);
  if (pl < lanes) {
    const float a4[4] = {sa[c], sa[c + 1], sa[c + 2], sa[c + 3]}, b4[4] = {sb[c], sb[c + 1], sb[c + 2], sb[c + 3]};
    const float r4[4] = {srs[c], srs[c + 1], srs[c + 2], srs[c + 3]}, m4[4] = {smu[c], smu[c + 1], smu[c + 2], smu[c + 3]};
    for (int pix = p0 + pl; pix < p1; pix += lanes) {
      const size_t off = ((size_t)n * p.HW + pix) * p.C + c;
      const float4 xv = __ldg(reinterpret_cast<const float4*>(p.x + off));
      const float4 gv = __ldg(reinterpret_cast<const float4*>(p.gy + off));
      const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs_[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float z = fmaf(a4[k], xs[k], b4[k]);
        const float gz = p.act ? gs_[k] * dsilu_f(z) : gs_[k];
        A[k] += gz;
        Bm[k] += gz * ((xs[k] - m4[k]) * r4[k]);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) { red[threadIdx.x][k] = A[k]; red[threadIdx.x][4 + k] = Bm[k]; }
  __syncthreads();
  if ((int)threadIdx.x < p.C) {   // thread = channel: sum over the pixel lanes in a fixed order
    const int cc = threadIdx.x, q4 = cc >> 2, k = cc & 3;
    float a = 0.f, b = 0.f;
    for (int l = 0; l < lanes; ++l) { a += red[l * L4 + q4][k]; b += red[l * L4 + q4][4 + k]; }
    atomicAdd(p.sumA + (size_t)n * p.sum_stride + cc, a);
    atomicAdd(p.sumB + (size_t)n * p.sum_stride + cc, b);
  }
}

__global__ void __launch_bounds__(kNormThreads) norm_bwd_pass2_kernel(const NormBwdParams p, int ppb) {
  __shared__ float sa[kMaxCin], sb[kMaxCin], sk[kMaxCin], srs[kMaxCin], smu[kMaxCin];
  __shared__ float sm1[8], sm2[8];
  const int n = blockIdx.y;
  norm_coeffs(p, n, sa, sb, sk, srs, smu);
  const int G = p.C / p.gs;
  if ((int)threadIdx.x < G) {
    float m1 = 0.f, m2 = 0.f;
    for (int c = threadIdx.x * p.gs; c < (threadIdx.x + 1) * p.gs; ++c) {
      m1 += sk[c] * p.sumA[(size_t)n * p.sum_stride + c];
      m2 += sk[c] * p.sumB[(size_t)n * p.sum_stride + c];
    }
    const float cnt = (float)p.HW * p.gs;
    sm1[threadIdx.x] = m1 / cnt;
    sm2[threadIdx.x] = m2 / cnt;
  }
  __syncthreads();
  const int L4 = p.C >> 2, lanes = kNormThreads / L4;
  const int c4 = threadIdx.x % L4, pl = threadIdx.x / L4;
  const int c = c4 * 4;
  if (pl >= lanes) return;
  const float a4[4] = {sa[c], sa[c + 1], sa[c + 2], sa[c + 3]}, b4[4] = {sb[c], sb[c + 1], sb[c + 2], sb[c + 3]};
  const float r4[4] = {srs[c], srs[c + 1], srs[c + 2], srs[c + 3]}, m4[4] = {smu[c], smu[c + 1], smu[c + 2], smu[c + 3]};
  const float k4[4] = {sk[c], sk[c + 1], sk[c + 2], sk[c + 3]};
  const float m1 = sm1[c / p.gs], m2 = sm2[c / p.gs];   // a channel quad never straddles a group (gs multiple of 4)
  const int p0 = blockIdx.x * ppb, p1 = min(p0 + ppb, p.HW);
  for (int pix = p0 + pl; pix < p1; pix += lanes) {
    const size_t off = ((size_t)n * p.HW + pix) * p.C + c;
    const float4 xv = __ldg(reinterpret_cast<const float4*>(p.x + off));
    const float4 gv = __ldg(reinterpret_cast<const float4*>(p.gy + off));
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w}, gs_[4] = {gv.x, gv.y, gv.z, gv.w};
    float o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float z = fmaf(a4[k], xs[k], b4[k]);
      const float gz = p.act ? gs_[k] * dsilu_f(z) : gs_[k];
      const float xhat = (xs[k] - m4[k]) * r4[k];
      o[k] = r4[k] * (k4[k] * gz - m1 - xhat * m2);
    }
    float4 ov = make_float4(o[0], o[1], o[2], o[3]);
    if (p.addend) { const float4 av = __ldg(reinterpret_cast<const float4*>(p.addend + off)); ov.x += av.x; ov.y += av.y; ov.z += av.z; ov.w += av.w; }
    float4* dst = reinterpret_cast<float4*>(p.gx + off);
    if (p.accumulate) { const float4 d = *dst; ov.x += d.x; ov.y += d.y; ov.z += d.z; ov.w += d.w; }
    *dst = ov;
  }
}

// d gamma[c] += alpha * sum_n sumB[n][c],  d beta[c] += alpha * sum_n sumA[n][c]   (affine GroupNorm parameters)
__global__ void affine_param_grad_kernel(const float* __restrict__ sumA, const float* __restrict__ sumB, int B, int C, int stride,
                                         float* __restrict__ dgamma, float* __restrict__ dbeta, const float* __restrict__ inv_scale) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float a = 0.f, b = 0.f;
  for (int n = 0; n < B; ++n) { a += sumA[(size_t)n * stride + c]; b += sumB[(size_t)n * stride + c]; }
  const float s = inv_scale ? *inv_scale : 1.f;
  dgamma[c] += b * s;
  dbeta[c] += a * s;
}

// ------------------------------------------------------------------------------------------------ elementwise adjoints
// nearest-2x upsample adjoint (blocks.py:109): out[n][y][x][c] (+)= sum of the 2x2 block of in[n][2y+dy][2x+dx][c]
__global__ void sumpool2_kernel(const float* __restrict__ in, float* __restrict__ out, int H, int W, int C, int accumulate, long long total4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // float4 index into out [B][H][W][C]
  if (i >= total4) return;
  const int L4 = C >> 2;
  const int c4 = (int)(i % L4);
  const long long pix = i / L4;
  const int x = (int)(pix % W);
  const long long r = pix / W;
  const int y = (int)(r % H);
  const long long n = r / H;
  const float4* src = reinterpret_cast<const float4*>(in) + (((n * 2 * H + 2 * y) * 2 * W) + 2 * x) * L4 + c4;
  const float4 a = __ldg(src), b = __ldg(src + L4), c = __ldg(src + (size_t)2 * W * L4), d = __ldg(src + (size_t)2 * W * L4 + L4);
  float4 o = make_float4((a.x + b.x) + (c.x + d.x), (a.y + b.y) + (c.y + d.y), (a.z + b.z) + (c.z + d.z), (a.w + b.w) + (c.w + d.w));
  float4* dst = reinterpret_cast<float4*>(out) + i;
  if (accumulate) { const float4 v = *dst; o.x += v.x; o.y += v.y; o.z += v.z; o.w += v.w; }
  *dst = o;
}
// dpre = dh * silu'(pre)   (cond_proj SiLU, inner_model.py:33)
__global__ void dsilu_mul_kernel(const float* __restrict__ pre, const float* __restrict__ dh, float* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = dh[i] * dsilu_f(pre[i]);
}

// ------------------------------------------------------------------------------------------------ small SGEMM
// C[m][n] (+)= alpha * sum_k A(m,k) * B(k,n),   A(m,k) = A[m*sam + k*sak],  B(k,n) = B[k*sbk + n*sbn]   (fp32, any strides)
// 64x64 tiles, 16-deep K slices, 256 threads x (4x4) outputs.  Used for every nn.Linear backward on the path
// (blocks.py:39 FiLM, inner_model.py:31-35 cond_proj, actor_critic.py:46-48 LSTMCell / heads).
__global__ void __launch_bounds__(256) sgemm_kernel(const float* __restrict__ A, long long sam, long long sak,
                                                    const float* __restrict__ Bm, long long sbk, long long sbn,
                                                    float* __restrict__ C, long long ldc, int M, int N, int K,
                                                    const float* __restrict__ alpha_ptr, int accumulate,
                                                    int kchunk = 0, long long c_split_stride = 0) {
  __shared__ float As[16][64 + 4], Bs[16][64 + 4];
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  // split-K (gridDim.z > 1): block z multiplies the K range [z * kchunk, (z + 1) * kchunk) into its own partial C at
  // C + z * c_split_stride; splitk_reduce_kernel then adds the partials in a fixed order (deterministic)
  const int kbeg = kchunk > 0 ? blockIdx.z * kchunk : 0;
  if (kchunk > 0) { K = min(K, kbeg + kchunk); C += (long long)blockIdx.z * c_split_stride; }
  float acc[4][4] = {};
  for (int k0 = kbeg; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      // choose the fast index along the contiguous dimension of each operand
      int kk, mm;
      if (sak == 1) { kk = i & 15; mm = i >> 4; } else { mm = i & 63; kk = i >> 6; }
      As[kk][mm] = (m0 + mm < M && k0 + kk < K) ? A[(long long)(m0 + mm) * sam + (long long)(k0 + kk) * sak] : 0.f;
      int kb, nn;
      if (sbk == 1) { kb = i & 15; nn = i >> 4; } else { nn = i & 63; kb = i >> 6; }
      Bs[kb][nn] = (n0 + nn < N && k0 + kb < K) ? Bm[(long long)(k0 + kb) * sbk + (long long)(n0 + nn) * sbn] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  const float alpha = alpha_ptr ? *alpha_ptr : 1.f;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
      if (m < M && n < N) {
        float* c = C + (long long)m * ldc + n;
        const float v = alpha * acc[i][j];
        *c = accumulate ? *c + v : v;
      }
    }
}

// out[i] (+)= alpha * sum_z partial[z][i], z ascending (the second half of a split-K sgemm)
__global__ void splitk_reduce_kernel(const float* __restrict__ partial, int splits, long long count, float* __restrict__ out,
                                     const float* __restrict__ alpha_ptr, int accumulate) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  float s = 0.f;
  for (int z = 0; z < splits; ++z) s += partial[(long long)z * count + i];
  if (alpha_ptr) s *= *alpha_ptr;
  out[i] = accumulate ? out[i] + s : s;
}

// FiLM weight gradients through a row-pointer table: the 44 AdaGroupNorm.linear layers (blocks.py:39) were batched into one
// [film_rows][CC] matrix for the forward; their gradients go back to 44 separate parameters.
//   dW_row[f][k] += alpha * sum_n dfilm[n][f] * cond[n][k] ;  db_row[f] += alpha * sum_n dfilm[n][f]
// grid (film_rows / 8, ceil(CC / 256)), 256 threads = the 256 cond columns of slice blockIdx.y (kSlices = false: CC <= 256, one
// slice); the first 8 threads of slice 0 also sum the biases.  Each sum runs over n ascending whatever CC is.  woff[f] / boff[f]
// are offsets into the flat gradient buffer.
template <bool kSlices>
__global__ void __launch_bounds__(256) film_wgrad_kernel(const float* __restrict__ dfilm, const float* __restrict__ cond,
                                                         float* __restrict__ grads, const long long* __restrict__ woff,
                                                         const long long* __restrict__ boff, int B, int rows, int CC,
                                                         const float* __restrict__ inv_scale) {
  __shared__ float sd[8][64];
  const int f0 = blockIdx.x * 8, k = (kSlices ? blockIdx.y * 256 : 0) + threadIdx.x;   // k < 8: a bias row (slice 0)
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float bsum = 0.f;
  for (int nb = 0; nb < B; nb += 64) {
    __syncthreads();
    for (int i = threadIdx.x; i < 8 * 64; i += 256) {
      const int r = i >> 6, nn = i & 63;
      sd[r][nn] = (nb + nn < B && f0 + r < rows) ? dfilm[(size_t)(nb + nn) * rows + f0 + r] : 0.f;
    }
    __syncthreads();
    const int lim = min(64, B - nb);
    if (k < CC) {
      for (int nn = 0; nn < lim; ++nn) {
        const float cv = __ldg(cond + (size_t)(nb + nn) * CC + k);
#pragma unroll
        for (int r = 0; r < 8; ++r) acc[r] = fmaf(sd[r][nn], cv, acc[r]);
      }
    }
    if (k < 8) for (int nn = 0; nn < lim; ++nn) bsum += sd[k][nn];
  }
  const float s = inv_scale ? *inv_scale : 1.f;
  if (k < CC) {
#pragma unroll
    for (int r = 0; r < 8; ++r) if (f0 + r < rows) grads[woff[f0 + r] + k] += acc[r] * s;
  }
  if (k < 8 && f0 + k < rows) grads[boff[f0 + k]] += bsum * s;
}

// act_emb gradient (inner_model.py:27-30,45): dE[a][j] += alpha * de[n][t*E + j] for a = act[n][t]
__global__ void embedding_bwd_kernel(const float* __restrict__ de, const int64_t* __restrict__ act, float* __restrict__ dE,
                                     int B, int CC, int T, int num_actions, const float* __restrict__ inv_scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * CC) return;
  const int n = i / CC, k = i - n * CC, E = CC / T;
  long long a = act[(size_t)n * T + k / E];
  a = a < 0 ? 0 : (a >= num_actions ? num_actions - 1 : a);
  atomicAdd(dE + (size_t)a * E + (k % E), de[i] * (inv_scale ? *inv_scale : 1.f));
}

// ------------------------------------------------------------------------------------------------ deterministic arms
// What torch.use_deterministic_algorithms selects in place of the fp32 atomics above: every sum has one owner and a fixed order.

// colsum_kernel's row chunks, each block's column sums stored (unscaled) to part[blockIdx.x][C] instead of added to `out`
__global__ void __launch_bounds__(256) colsum_part_kernel(const float* __restrict__ x, float* __restrict__ part, long long rows, int C) {
  __shared__ float cs_sm[1024];
  const int cbase = blockIdx.y * 256;
  const int Cb = min(256, C - cbase);
  const int L4 = Cb >> 2;
  const int lanes = 256 / L4;
  const int c4 = threadIdx.x % L4, rl = threadIdx.x / L4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (rl < lanes) {
    for (long long r = (long long)blockIdx.x * lanes + rl; r < rows; r += (long long)gridDim.x * lanes) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * C + cbase) + c4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    reinterpret_cast<float4*>(cs_sm + (size_t)rl * Cb)[c4] = acc;
  }
  __syncthreads();
  if ((int)threadIdx.x < Cb) {
    float s = 0.f;
    for (int k = 0; k < lanes; ++k) s += cs_sm[(size_t)k * Cb + threadIdx.x];
    part[(size_t)blockIdx.x * C + cbase + threadIdx.x] = s;
  }
}
// out[c] (and out2[c]) += inv_scale * sum over the nparts block sums of part, in block order
__global__ void colsum_reduce_kernel(const float* __restrict__ part, int nparts, int C, int Creal, float* __restrict__ out,
                                     float* __restrict__ out2, const float* __restrict__ inv_scale) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= Creal) return;
  float s = 0.f;
  for (int b = 0; b < nparts; ++b) s += part[(size_t)b * C + c];
  s *= inv_scale ? *inv_scale : 1.f;
  out[c] += s;
  if (out2) out2[c] += s;
}

// embedding_bwd_kernel gathered: one thread per table entry (a, j) walks the batch rows and their T actions in order
__global__ void embedding_bwd_det_kernel(const float* __restrict__ de, const int64_t* __restrict__ act, float* __restrict__ dE,
                                         int B, int CC, int T, int num_actions, const float* __restrict__ inv_scale) {
  const int E = CC / T;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= num_actions * E) return;
  const int a = i / E, j = i - a * E;
  float s = 0.f;
  for (int n = 0; n < B; ++n)
    for (int t = 0; t < T; ++t) {
      long long an = act[(size_t)n * T + t];
      an = an < 0 ? 0 : (an >= num_actions ? num_actions - 1 : an);
      if (an == a) s += de[(size_t)n * CC + t * E + j] * (inv_scale ? *inv_scale : 1.f);
    }
  dE[i] += s;
}

// ------------------------------------------------------------------------------------------------ attention backward
// SelfAttention2d (blocks.py:51-72) backward, one CTA per image (L <= 64 tokens, C in {32, 64}, head_dim 8).  kL = 64: the
// token count is a compile-time constant (the 8x8 level of a 64x64 frame); kL = 0: any L from 1 to 64, read from p.L, the same
// arithmetic in the same order.  The forward is recomputed in shared memory (normed x, qkv, per-row softmax statistics), then:
//   out = xn + Wo y + bo              ->  g_xn = g_out,  g_y = Wo^T g_out,  dWo += g_out (x) y,  dbo += sum g_out
//   y = P v, P = softmax(q k^T / sqrt d)  ->  g_v = P^T g_y,  g_s = P o (g_y v^T - rowsum(P o g_y v^T)),  g_q = g_s k / sqrt d,
//                                             g_k = g_s^T q / sqrt d
//   qkv = Wqkv xn + b                 ->  dWqkv += g_qkv (x) xn,  dbqkv += sum g_qkv,  g_xn += Wqkv^T g_qkv
//   xn = GroupNorm(x)                 ->  d gamma, d beta, g_x  (two group means)
// Parameter gradients are accumulated with fp32 atomics (scaled by inv_scale); g_x is written (assigned) to gx.
struct AttnBwdParams {
  const float* x; const double* st_in; const float* gamma; const float* beta;
  const float* wqkv; const float* bqkv; const float* wout;
  const float* gout;     // NHWC [B][L][C] gradient wrt the attention output
  float* gx;             // NHWC [B][L][C] gradient wrt the attention input (assigned)
  float *dgamma, *dbeta, *dwqkv, *dbqkv, *dwout, *dbout;
  const float* inv_scale;
  int L, C, gs;
  float eps;
};

template <int C, int kL>
__global__ void __launch_bounds__(kAttnThreads) attn_bwd_kernel(const AttnBwdParams p) {
  static_assert(kL == kAttnL || kL == 0, "attn_bwd_kernel: kL is 64 or 0 (runtime token count)");
  constexpr int C3 = 3 * C, XP = C + 1, QP = C3 + 4, HEADS = C / 8;
  const int L = kL ? kL : p.L;
  extern __shared__ __align__(16) float sm_ab[];
  float* xh = sm_ab;              // [L][XP]  xhat = (x - mean) * rstd
  float* qkv = xh + L * XP;       // [L][QP]
  float* ys = qkv + L * QP;       // [L][XP]  attention output y (pre out_proj)
  float* gys = ys + L * XP;       // [L][XP]  g_y
  float* gqkv = gys + L * XP;     // [L][QP]  g_qkv
  float* gxn = gqkv + L * QP;     // [L][XP]  g_xn (starts as g_out)
  float* rowst = gxn + L * XP;    // [HEADS*L][3]  (max, 1/den, D)
  __shared__ float s_rstd[4], s_g1[4], s_g2[4];
  const int n = blockIdx.x, tid = threadIdx.x;
  const int G = C / p.gs;
  const float alpha = p.inv_scale ? *p.inv_scale : 1.f;
  const float* xg = p.x + (size_t)n * L * C;
  const float* gg = p.gout + (size_t)n * L * C;
  if (tid < G) {
    const double cnt = (double)L * p.gs;
    const double mean = p.st_in[((size_t)n * G + tid) * 2] / cnt;
    double var = p.st_in[((size_t)n * G + tid) * 2 + 1] / cnt - mean * mean;
    var = var > 0.0 ? var : 0.0;
    s_g1[tid] = (float)mean;
    s_rstd[tid] = (float)(1.0 / sqrt(var + (double)p.eps));
  }
  __syncthreads();
  for (int i = tid; i < L * C; i += kAttnThreads) {
    const int l = i / C, c = i - l * C, g = c / p.gs;
    xh[l * XP + c] = (xg[i] - s_g1[g]) * s_rstd[g];
    gxn[l * XP + c] = gg[i];
  }
  __syncthreads();
  // ---- qkv = Wqkv xn + b   (xn = xhat * gamma + beta); item (token l, output group og): at L = 64 one per thread
  {
    constexpr int NG = kAttnThreads / kAttnL, NO = C3 / NG;
    auto project = [&](int l, int og) {
      float acc[NO];
#pragma unroll
      for (int i = 0; i < NO; ++i) acc[i] = __ldg(p.bqkv + og * NO + i);
      for (int c = 0; c < C; ++c) {
        const float xn = fmaf(xh[l * XP + c], __ldg(p.gamma + c), __ldg(p.beta + c));
#pragma unroll
        for (int i = 0; i < NO; ++i) acc[i] = fmaf(__ldg(p.wqkv + (size_t)(og * NO + i) * C + c), xn, acc[i]);
      }
#pragma unroll
      for (int i = 0; i < NO; ++i) qkv[l * QP + og * NO + i] = acc[i];
    };
    if (kL) project(tid % L, tid / L);
    else for (int it = tid; it < L * NG; it += kAttnThreads) project(it % L, it / L);
  }
  __syncthreads();
  // ---- pass A1: softmax row statistics and y, item = (head, query)
  for (int it = tid; it < HEADS * L; it += kAttnThreads) {
    const int h = it / L, l = it - h * L;
    float q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) q[e] = qkv[l * QP + h * 8 + e] * 0.35355339059327373f;
    float mx = -INFINITY;
    for (int j = 0; j < L; ++j) {
      float sj = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) sj = fmaf(q[e], qkv[j * QP + C + h * 8 + e], sj);
      mx = fmaxf(mx, sj);
    }
    float den = 0.f, y[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < L; ++j) {
      float sj = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) sj = fmaf(q[e], qkv[j * QP + C + h * 8 + e], sj);
      const float pj = expf(sj - mx);
      den += pj;
#pragma unroll
      for (int e = 0; e < 8; ++e) y[e] = fmaf(pj, qkv[j * QP + 2 * C + h * 8 + e], y[e]);
    }
    const float inv = 1.f / den;
#pragma unroll
    for (int e = 0; e < 8; ++e) ys[l * XP + h * 8 + e] = y[e] * inv;
    rowst[it * 3] = mx; rowst[it * 3 + 1] = inv;
  }
  __syncthreads();
  // ---- out_proj backward: g_y = Wo^T g_out ; dWo, dbo
  for (int i = tid; i < L * C; i += kAttnThreads) {
    const int l = i / C, c = i - l * C;
    float a = 0.f;
    for (int o = 0; o < C; ++o) a = fmaf(gxn[l * XP + o], __ldg(p.wout + (size_t)o * C + c), a);
    gys[l * XP + c] = a;
  }
  for (int i = tid; i < C * C; i += kAttnThreads) {
    const int o = i / C, c = i - o * C;
    float a = 0.f;
    for (int l = 0; l < L; ++l) a = fmaf(gxn[l * XP + o], ys[l * XP + c], a);
    atomicAdd(p.dwout + i, a * alpha);
  }
  if (tid < C) {
    float a = 0.f;
    for (int l = 0; l < L; ++l) a += gxn[l * XP + tid];
    atomicAdd(p.dbout + tid, a * alpha);
  }
  __syncthreads();
  // ---- pass A2: D = sum_j P (g_y . v_j) and g_q, item = (head, query)
  for (int it = tid; it < HEADS * L; it += kAttnThreads) {
    const int h = it / L, l = it - h * L;
    float q[8], gy[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { q[e] = qkv[l * QP + h * 8 + e] * 0.35355339059327373f; gy[e] = gys[l * XP + h * 8 + e]; }
    const float mx = rowst[it * 3], inv = rowst[it * 3 + 1];
    float D = 0.f;
    for (int j = 0; j < L; ++j) {
      float sj = 0.f, ga = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) { sj = fmaf(q[e], qkv[j * QP + C + h * 8 + e], sj); ga = fmaf(gy[e], qkv[j * QP + 2 * C + h * 8 + e], ga); }
      D = fmaf(expf(sj - mx) * inv, ga, D);
    }
    float gq[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < L; ++j) {
      float sj = 0.f, ga = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) { sj = fmaf(q[e], qkv[j * QP + C + h * 8 + e], sj); ga = fmaf(gy[e], qkv[j * QP + 2 * C + h * 8 + e], ga); }
      const float gs = expf(sj - mx) * inv * (ga - D);
#pragma unroll
      for (int e = 0; e < 8; ++e) gq[e] = fmaf(gs, qkv[j * QP + C + h * 8 + e], gq[e]);
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) gqkv[l * QP + h * 8 + e] = gq[e] * 0.35355339059327373f;
    rowst[it * 3 + 2] = D;
  }
  __syncthreads();
  // ---- pass B: g_k and g_v, item = (head, key)
  for (int it = tid; it < HEADS * L; it += kAttnThreads) {
    const int h = it / L, j = it - h * L;
    float k[8], v[8], gk[8] = {0, 0, 0, 0, 0, 0, 0, 0}, gv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
    for (int e = 0; e < 8; ++e) { k[e] = qkv[j * QP + C + h * 8 + e]; v[e] = qkv[j * QP + 2 * C + h * 8 + e]; }
    for (int l = 0; l < L; ++l) {
      const float mx = rowst[(h * L + l) * 3], inv = rowst[(h * L + l) * 3 + 1], D = rowst[(h * L + l) * 3 + 2];
      float sj = 0.f, ga = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        sj = fmaf(qkv[l * QP + h * 8 + e] * 0.35355339059327373f, k[e], sj);
        ga = fmaf(gys[l * XP + h * 8 + e], v[e], ga);
      }
      const float pj = expf(sj - mx) * inv;
      const float gs = pj * (ga - D);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        gk[e] = fmaf(gs, qkv[l * QP + h * 8 + e] * 0.35355339059327373f, gk[e]);
        gv[e] = fmaf(pj, gys[l * XP + h * 8 + e], gv[e]);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) { gqkv[j * QP + C + h * 8 + e] = gk[e]; gqkv[j * QP + 2 * C + h * 8 + e] = gv[e]; }
  }
  __syncthreads();
  // ---- qkv projection backward: dWqkv, dbqkv, g_xn += Wqkv^T g_qkv
  for (int i = tid; i < C3 * C; i += kAttnThreads) {
    const int o = i / C, c = i - o * C;
    const float ga = __ldg(p.gamma + c), be = __ldg(p.beta + c);
    float a = 0.f;
    for (int l = 0; l < L; ++l) a = fmaf(gqkv[l * QP + o], fmaf(xh[l * XP + c], ga, be), a);
    atomicAdd(p.dwqkv + i, a * alpha);
  }
  if (tid < C3) {
    float a = 0.f;
    for (int l = 0; l < L; ++l) a += gqkv[l * QP + tid];
    atomicAdd(p.dbqkv + tid, a * alpha);
  }
  for (int i = tid; i < L * C; i += kAttnThreads) {
    const int l = i / C, c = i - l * C;
    float a = gxn[l * XP + c];
    for (int o = 0; o < C3; ++o) a = fmaf(gqkv[l * QP + o], __ldg(p.wqkv + (size_t)o * C + c), a);
    gys[l * XP + c] = a;           // g_xn complete (gys is free now)
  }
  __syncthreads();
  // ---- GroupNorm backward (affine)
  float* const red = kL ? ys : qkv;   // two rows of per-channel sums: ys holds only one at L = 1, qkv is free as well
  if (tid < C) {
    float a = 0.f, b = 0.f;
    for (int l = 0; l < L; ++l) { const float g = gys[l * XP + tid]; a += g; b += g * xh[l * XP + tid]; }
    atomicAdd(p.dbeta + tid, a * alpha);
    atomicAdd(p.dgamma + tid, b * alpha);
    const float ga = __ldg(p.gamma + tid);
    red[tid] = ga * a;             // per-channel sums of g_xhat and g_xhat * xhat (ys is free now)
    red[XP + tid] = ga * b;
  }
  __syncthreads();
  if (tid < G) {
    float m1 = 0.f, m2 = 0.f;
    for (int c = tid * p.gs; c < (tid + 1) * p.gs; ++c) { m1 += red[c]; m2 += red[XP + c]; }
    const float cnt = (float)L * p.gs;
    s_g1[tid] = m1 / cnt; s_g2[tid] = m2 / cnt;
  }
  __syncthreads();
  float* gxo = p.gx + (size_t)n * L * C;
  for (int i = tid; i < L * C; i += kAttnThreads) {
    const int l = i / C, c = i - l * C, g = c / p.gs;
    gxo[i] = s_rstd[g] * (__ldg(p.gamma + c) * gys[l * XP + c] - s_g1[g] - xh[l * XP + c] * s_g2[g]);
  }
}

// ------------------------------------------------------------------------------------------------ actor-critic pieces
// MaxPool2d(2) backward (actor_critic.py:109): the gradient of a pooled element goes to the window position that holds the
// maximum (the first one in window order on an exact tie, like ATen).  y: pre-pool NHWC [B][H][W][C]; gp: NHWC
// [B][H/2][W/2][C], floor division: at an odd H (W) the last row (column) is in no window, and the threads of the last window
// row (column) write its zero gradient.
__global__ void maxpool2_bwd_kernel(const float* __restrict__ y, const float* __restrict__ gp, float* __restrict__ gy, int H, int W, int C) {
  const int n = blockIdx.y;
  const int Ho = H >> 1, Wo = W >> 1;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Ho * Wo * C) return;
  const int c = i % C, pix = i / C, xo = pix % Wo, yo = pix / Wo;
  const size_t base = (((size_t)n * H + 2 * yo) * W + 2 * xo) * C + c;
  const size_t o[4] = {base, base + C, base + (size_t)W * C, base + (size_t)W * C + C};
  const float v[4] = {y[o[0]], y[o[1]], y[o[2]], y[o[3]]};
  int am = 0;
#pragma unroll
  for (int k = 1; k < 4; ++k) if (v[k] > v[am]) am = k;
  const float g = gp[(size_t)n * Ho * Wo * C + i];
#pragma unroll
  for (int k = 0; k < 4; ++k) gy[o[k]] = k == am ? g : 0.f;
  const bool last_col = (W & 1) && xo == Wo - 1, last_row = (H & 1) && yo == Ho - 1;
  if (last_col) { gy[base + 2 * C] = 0.f; gy[base + (size_t)W * C + 2 * C] = 0.f; }
  if (last_row) { gy[base + (size_t)2 * W * C] = 0.f; gy[base + (size_t)2 * W * C + C] = 0.f; }
  if (last_col && last_row) gy[base + (size_t)2 * W * C + 2 * C] = 0.f;
}

// LSTMCell backward (actor_critic.py:46,72; torch gate order i, f, g, o).  gates: pre-activations [B][4H] of the forward;
// g_h, g_c: gradients wrt the new hidden / cell state (g_c may be null); outputs dgates [B][4H] and g_c_in [B][H].
__global__ void lstm_cell_bwd_kernel(const float* __restrict__ gates, const float* __restrict__ c_in, const float* __restrict__ g_h,
                                     const float* __restrict__ g_c, float* __restrict__ dgates, float* __restrict__ g_c_in, int B, int Hd) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * Hd) return;
  const int n = idx / Hd, j = idx - n * Hd;
  const float* g = gates + (size_t)n * 4 * Hd;
  const float ig = 1.f / (1.f + expf(-g[j])), fg = 1.f / (1.f + expf(-g[Hd + j]));
  const float gg = tanhf(g[2 * Hd + j]), og = 1.f / (1.f + expf(-g[3 * Hd + j]));
  const float c = fg * c_in[idx] + ig * gg;
  const float tc = tanhf(c);
  const float gh = g_h ? g_h[idx] : 0.f;
  const float gc = (g_c ? g_c[idx] : 0.f) + gh * og * (1.f - tc * tc);
  float* d = dgates + (size_t)n * 4 * Hd;
  d[j] = gc * gg * ig * (1.f - ig);
  d[Hd + j] = gc * c_in[idx] * fg * (1.f - fg);
  d[2 * Hd + j] = gc * ig * (1.f - gg * gg);
  d[3 * Hd + j] = gh * tc * og * (1.f - og);
  g_c_in[idx] = gc * fg;
}

// g_h[n][j] = g_hx[n][j] + sum_a g_logits[n][a] Wa[a][j] + g_val[n] Wc[j]     (actor / critic heads, actor_critic.py:73)
__global__ void heads_bwd_kernel(const float* __restrict__ g_hx, const float* __restrict__ g_logits, const float* __restrict__ g_val,
                                 const float* __restrict__ Wa, const float* __restrict__ Wc, float* __restrict__ g_h, int B, int Hd, int A) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * Hd) return;
  const int n = idx / Hd, j = idx - n * Hd;
  float a = g_hx ? g_hx[idx] : 0.f;
  if (g_logits) for (int k = 0; k < A; ++k) a = fmaf(g_logits[(size_t)n * A + k], Wa[(size_t)k * Hd + j], a);
  if (g_val) a = fmaf(g_val[n], Wc[j], a);
  g_h[idx] = a;
}
// out[j] += sum_n a[n] * b[n][j]  and  out_b += sum_n a[n]   (critic head: dWc, dbc)
__global__ void vec_outer_sum_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, float* __restrict__ out_b, int B, int Hd) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < Hd) {
    float s = 0.f;
    for (int n = 0; n < B; ++n) s = fmaf(a[n], b[(size_t)n * Hd + j], s);
    out[j] += s;
  }
  if (j == 0) { float s = 0.f; for (int n = 0; n < B; ++n) s += a[n]; *out_b += s; }
}
// out[c] += sum_rows x[row][c] for a small [rows][C] matrix (actor bias; C = num_actions)
__global__ void small_colsum_kernel(const float* __restrict__ x, int rows, int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int r = 0; r < rows; ++r) s += x[(size_t)r * C + c];
  out[c] += s;
}
// x *= scale[0]   (the encoder gradient enters the fp16 tensor-core path scaled)
__global__ void scale_inplace_kernel(float* __restrict__ x, const float* __restrict__ scale, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] *= scale[0];
}

// ------------------------------------------------------------------------------------------------ lambda-returns
// compute_lambda_returns (actor_critic.py:116-143), one thread per environment walking time backwards.  fp32 operations in
// the reference's order with un-contracted multiplies / adds, so the result is bit-identical to the torch expression:
//   r = sign(rew);  ret[t] = r + (1-end) * gamma * ((1-trunc) * (1-lambda) + trunc) * vb[t]
//   ret[t] += (!(end|trunc)) * gamma * lambda * last ;  last = ret[t]          (last starts at vb[T-1])
// rew / vb fp32 [B][T]; end / trunc int64 [B][T]; ret fp32 [B][T].
__global__ void lambda_returns_kernel(const float* __restrict__ rew, const long long* __restrict__ end, const long long* __restrict__ trunc,
                                      const float* __restrict__ vb, float* __restrict__ ret, int B, int T, float gamma, float lambda_,
                                      float one_minus_lambda) {   // (1 - lambda) is evaluated in DOUBLE by python, then rounded: host passes it
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= B) return;
  float last = vb[(size_t)n * T + T - 1];
  for (int t = T - 1; t >= 0; --t) {
    const size_t i = (size_t)n * T + t;
    const float r = (float)(rew[i] > 0.f) - (float)(rew[i] < 0.f);              // torch.sign
    const float e = (float)end[i], tr = (float)trunc[i];
    const float not_end = 1.f - e, not_trunc = 1.f - tr;
    // not_end * gamma * (not_trunc * (1 - lambda) + trunc) * vb
    const float inner = __fadd_rn(__fmul_rn(not_trunc, one_minus_lambda), tr);
    float v = __fadd_rn(r, __fmul_rn(__fmul_rn(__fmul_rn(not_end, gamma), inner), vb[i]));
    if (lambda_ != 0.f) {
      const float alive = (e + tr) >= 1.f ? 0.f : 1.f;
      v = __fadd_rn(v, __fmul_rn(__fmul_rn(__fmul_rn(alive, gamma), lambda_), last));
      last = v;
    }
    ret[i] = v;
  }
}

// ------------------------------------------------------------------------------------------------ transposed weight packing
// dgrad = the forward implicit GEMM on dL/dy with weights transposed and taps flipped (tests/test_gpu_conv.py dgrad case):
//   w'[co' = ci][ci' = co][t'] = w[co][ci_off + ci][taps - 1 - t']       packed [tap][CinP/8][CoutP][8] fp16
// where CinP = round16(Cout_fwd) channels of the gradient operand and CoutP = round16(Cin_k) outputs.
__global__ void pack_conv_weight_T_kernel(const float* __restrict__ w, __half* __restrict__ wpk, int CoutF, int CinTotF,
                                          int ci_off, int CinK, int CinP, int CoutP, int taps) {
  const int total = taps * CinP * CoutP;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int e = i & 7;
    const int cop = (i >> 3) % CoutP;              // output channel of the dgrad conv = forward input channel
    const int j = (i >> 3) / CoutP % (CinP >> 3);
    const int t = (i >> 3) / CoutP / (CinP >> 3);
    const int cip = j * 8 + e;                     // input channel of the dgrad conv = forward output channel
    float v = 0.f;
    if (cop < CinK && cip < CoutF) v = w[((size_t)cip * CinTotF + ci_off + cop) * taps + (taps - 1 - t)];
    wpk[i] = __float2half_rn(v);
  }
}

// ------------------------------------------------------------------------------------------------ attention backward, C = 128
// At C = 128 the one-CTA backward above would need 343 KB of shared memory, so it is split (api.cu BwdBuilder::attn_split):
// attn_qkv_kernel<128> recomputes q | k | v into scratch ([B][3][16][64][8], head-major), attn_xn_kernel the normed input,
// sgemm gives g_y = g_out Wo, then attn_core_bwd_kernel runs one CTA per (head, image) and the projection gradients and
// g_xn += g_qkv Wqkv are sgemm / colsum launches, the GroupNorm backward the two-pass norm backward without SiLU.

// xn = GroupNorm(x) (gamma, beta) from the producer's statistics, NHWC [B][L][C] -> [B][L][C]
__global__ void attn_xn_kernel(const float* __restrict__ x, const double* __restrict__ st_in, const float* __restrict__ gamma,
                               const float* __restrict__ beta, float* __restrict__ xn, int L, int C, int gs, float eps, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = (int)(i % C);
  const long long n = i / ((long long)L * C);
  const int G = C / gs, g = c / gs;
  const double cnt = (double)L * gs;
  const double mean = st_in[(n * G + g) * 2] / cnt;
  double var = st_in[(n * G + g) * 2 + 1] / cnt - mean * mean;
  var = var > 0.0 ? var : 0.0;
  xn[i] = (x[i] - (float)mean) * (float)(1.0 / sqrt(var + (double)eps)) * gamma[c] + beta[c];
}

// One CTA of kAttnL threads per (head h, image n), L <= 64 tokens, head_dim 8; thread i owns token i (threads i >= L only
// meet the barriers).  kL = 64: L is a compile-time constant; kL = 0: any L from 1 to 64, passed in Lrt.  In: qkv
// (attn_qkv_kernel layout), gy = g_y, gout = g_out (both NHWC [B][L][C]).  Out: y (attention output before out_proj, NHWC),
// gqkv ([B][L][3C], q | k | v rows as in Wqkv), gxn = g_out (head h's channels; the g_qkv Wqkv product is added to it
// afterwards).
//   P = softmax(q k^T / sqrt 8), y = P v, g_v = P^T g_y, g_s = P o (g_y v^T - rowsum(g_y o y)), g_q = g_s k / sqrt 8,
//   g_k = g_s^T q / sqrt 8
constexpr int kAttnCoreThreads = kAttnL;
template <int kL>
__global__ void __launch_bounds__(kAttnCoreThreads) attn_core_bwd_kernel(const float* __restrict__ qkv, const float* __restrict__ gy,
                                                                        const float* __restrict__ gout, float* __restrict__ y,
                                                                        float* __restrict__ gqkv, float* __restrict__ gxn, int C, int Lrt) {
  static_assert(kL == kAttnL || kL == 0, "attn_core_bwd_kernel: kL is 64 or 0 (runtime token count)");
  constexpr int LM = kAttnL, LP = LM + 1;
  const int L = kL ? kL : Lrt;
  __shared__ float q[LM][8], k[LM][8], v[LM][8], g[LM][8], P[LM][LP], S[LM][LP];
  const int h = blockIdx.x, n = blockIdx.y, i = threadIdx.x, HEADS = C / 8;
  const bool own = kL || i < L;
  const float* base = qkv + (size_t)n * 3 * C * L;
  const size_t row = ((size_t)n * L + i) * C + h * 8;
  if (own) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      q[i][e] = base[((size_t)h * L + i) * 8 + e];
      k[i][e] = base[((size_t)(HEADS + h) * L + i) * 8 + e];
      v[i][e] = base[((size_t)(2 * HEADS + h) * L + i) * 8 + e];
      g[i][e] = gy[row + e];
      gxn[row + e] = gout[row + e];
    }
  }
  __syncthreads();
  const float sc = 0.35355339059327373f;   // 1/sqrt(8)
  float gq[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (own) {
    // ---- row i: softmax, y_i, g_s row
    float mx = -INFINITY;
    for (int j = 0; j < L; ++j) {
      float s = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) s = fmaf(q[i][e] * sc, k[j][e], s);
      P[i][j] = s;
      mx = fmaxf(mx, s);
    }
    float den = 0.f;
    for (int j = 0; j < L; ++j) { const float pj = expf(P[i][j] - mx); P[i][j] = pj; den += pj; }
    const float inv = 1.f / den;
    float yi[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int j = 0; j < L; ++j) {
      const float pj = P[i][j] * inv;
      P[i][j] = pj;
#pragma unroll
      for (int e = 0; e < 8; ++e) yi[e] = fmaf(pj, v[j][e], yi[e]);
    }
    float D = 0.f;
#pragma unroll
    for (int e = 0; e < 8; ++e) { y[row + e] = yi[e]; D = fmaf(g[i][e], yi[e], D); }
    for (int j = 0; j < L; ++j) {
      float dp = 0.f;
#pragma unroll
      for (int e = 0; e < 8; ++e) dp = fmaf(g[i][e], v[j][e], dp);
      const float ds = P[i][j] * (dp - D) * sc;
      S[i][j] = ds;
#pragma unroll
      for (int e = 0; e < 8; ++e) gq[e] = fmaf(ds, k[j][e], gq[e]);
    }
  }
  __syncthreads();
  if (!own) return;
  // ---- column j = i: g_k, g_v
  float gk[8] = {0, 0, 0, 0, 0, 0, 0, 0}, gv[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int r = 0; r < L; ++r) {
    const float ds = S[r][i], pr = P[r][i];
#pragma unroll
    for (int e = 0; e < 8; ++e) { gk[e] = fmaf(ds, q[r][e], gk[e]); gv[e] = fmaf(pr, g[r][e], gv[e]); }
  }
  float* o = gqkv + ((size_t)n * L + i) * 3 * C + h * 8;
#pragma unroll
  for (int e = 0; e < 8; ++e) { o[e] = gq[e]; o[C + e] = gk[e]; o[2 * C + e] = gv[e]; }
}

}  // namespace dmd
