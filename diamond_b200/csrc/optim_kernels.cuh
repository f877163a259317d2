// Optimizer kernels: clip_grad_norm_ and AdamW (src/trainer.py:373-377, src/utils.py:164) over every tensor of a parameter
// list in one launch each.  The list travels as a kernel parameter (OptTable, < 32 764 bytes: CUDA >= 12.1 on sm_70+), one
// entry per tensor; tensor i owns blocks [block0[i], block0[i+1]) and every block a chunk of kOptChunk elements of it.
// HBM-bound: 4 bytes per element for the norm, 8 for the scale, 28 for AdamW.  No fast-math: every operation is the IEEE
// one torch's CUDA kernels perform, in their order, so the step reproduces torch.optim.AdamW(foreach=False) bit for bit
// wherever its kernels contract the same way.
#pragma once
#include <cuda_runtime.h>

namespace dmd {

constexpr int kOptMaxTensors = 512;     // per launch; longer lists take ceil(n / 512) launches
constexpr int kOptThreads = 256;
constexpr int kOptChunk = 16384;        // elements per block (a multiple of 4 * kOptThreads)

struct OptTable {
  int count;                            // tensors in this launch
  float* p[kOptMaxTensors];
  float* g[kOptMaxTensors];
  float* m[kOptMaxTensors];
  float* v[kOptMaxTensors];
  long long n[kOptMaxTensors];
  float decay[kOptMaxTensors];          // float(1 - lr * weight_decay); 1 when weight_decay == 0 (torch skips the mul_)
  int block0[kOptMaxTensors];
  unsigned char vec[kOptMaxTensors];    // every pointer the kernel touches is 16-byte aligned: float4 body, scalar tail
};
static_assert(sizeof(OptTable) <= 32764, "OptTable must fit the kernel-parameter limit");

// The scalars of one AdamW step, rounded to fp32 on the host exactly as torch passes its Python floats to its kernels.
struct AdamWScalars {
  float w1;           // lerp weight 1 - beta1
  float beta2;        // exp_avg_sq.mul_(beta2)
  float omb2;         // addcmul_ value 1 - beta2
  float inv_bc2s;     // 1 / sqrt(bias_correction2): torch divides by a CPU scalar as a multiply by its fp32 reciprocal
  float eps;
  float neg_step;     // addcdiv_ value -lr / bias_correction1
};

__device__ __forceinline__ int opt_locate(const OptTable& t, int b) {
  int lo = 0, hi = t.count - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (t.block0[mid] <= b) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Block-wide fp64 sum in a fixed order (per-thread partials, then shuffles, then warp 0): deterministic for a fixed launch.
__device__ __forceinline__ double opt_block_sum(double x) {
  __shared__ double red[kOptThreads / 32];
  for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = x;
  __syncthreads();
  if (threadIdx.x < 32) {
    x = threadIdx.x < kOptThreads / 32 ? red[threadIdx.x] : 0.0;
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
  }
  return x;   // valid in thread 0
}

// partial[part0 + block] = sum of g^2 over the block's chunk, in fp64 (a float's square is exact in a double).
__global__ void __launch_bounds__(kOptThreads) grad_sqnorm_kernel(const __grid_constant__ OptTable t, double* __restrict__ partial,
                                                                   int part0) {
  const int i = opt_locate(t, blockIdx.x);
  const long long lo = (long long)(blockIdx.x - t.block0[i]) * kOptChunk;
  const long long hi = min(t.n[i], lo + kOptChunk);
  const float* __restrict__ g = t.g[i];
  double acc = 0.0;
  long long j = lo + threadIdx.x;
  if (t.vec[i]) {
    const long long hi4 = lo + ((hi - lo) & ~3ll);
    const float4* g4 = reinterpret_cast<const float4*>(g);
#pragma unroll 4
    for (long long k = lo / 4 + threadIdx.x; k < hi4 / 4; k += kOptThreads) {
      const float4 x = __ldcs(g4 + k);
      acc += (double)x.x * x.x + (double)x.y * x.y + (double)x.z * x.z + (double)x.w * x.w;
    }
    j = hi4 + threadIdx.x;
  }
  for (; j < hi; j += kOptThreads) acc += (double)g[j] * g[j];
  acc = opt_block_sum(acc);
  if (threadIdx.x == 0) partial[part0 + blockIdx.x] = acc;
}

// One block: the partials summed in a fixed order; out[0] = total_norm (fp32), out[1] = min(1, max_norm / (total_norm + 1e-6))
// as torch's clip_grad_norm_ computes it: fp32 add, reciprocal, multiply by max_norm, clamp(max = 1) -- which keeps a NaN.
__global__ void __launch_bounds__(kOptThreads) grad_norm_finalize_kernel(const double* __restrict__ partial, int nparts, float max_norm,
                                                                         float* __restrict__ out) {
  double acc = 0.0;
  for (int k = threadIdx.x; k < nparts; k += kOptThreads) acc += partial[k];
  acc = opt_block_sum(acc);
  if (threadIdx.x == 0) {
    const float tn = (float)sqrt(acc);
    const float c = __fmul_rn(__fdiv_rn(1.0f, __fadd_rn(tn, 1e-6f)), max_norm);
    out[0] = tn;
    out[1] = c > 1.0f ? 1.0f : c;
  }
}

// g *= coef[0] in place (torch._foreach_mul_ by the clamped coefficient).  A coefficient of exactly 1 leaves every gradient as
// it is, so the blocks return without touching memory.
__global__ void __launch_bounds__(kOptThreads) grad_scale_kernel(const __grid_constant__ OptTable t, const float* __restrict__ coef) {
  const float c = *coef;
  if (c == 1.0f) return;
  const int i = opt_locate(t, blockIdx.x);
  const long long lo = (long long)(blockIdx.x - t.block0[i]) * kOptChunk;
  const long long hi = min(t.n[i], lo + kOptChunk);
  float* __restrict__ g = t.g[i];
  long long j = lo + threadIdx.x;
  if (t.vec[i]) {
    const long long hi4 = lo + ((hi - lo) & ~3ll);
    float4* g4 = reinterpret_cast<float4*>(g);
#pragma unroll 4
    for (long long k = lo / 4 + threadIdx.x; k < hi4 / 4; k += kOptThreads) {
      float4 x = g4[k];
      x.x = __fmul_rn(x.x, c); x.y = __fmul_rn(x.y, c); x.z = __fmul_rn(x.z, c); x.w = __fmul_rn(x.w, c);
      g4[k] = x;
    }
    j = hi4 + threadIdx.x;
  }
  for (; j < hi; j += kOptThreads) g[j] = __fmul_rn(g[j], c);
}

// torch 2.11 _single_tensor_adam with decoupled weight decay, one element; each line is one torch kernel, rounded to fp32
// between them, with the fused multiply-adds its CUDA functors compile to:
//   param.mul_(1 - lr*wd); exp_avg.lerp_(grad, 1 - beta1)            (two-branch lerp: weight < 0.5 ? s + w(e - s) : e - (e - s)(1 - w))
//   exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value = 1 - beta2)   (a + value * (b * c))
//   denom = (exp_avg_sq.sqrt() / bias_correction2_sqrt).add_(eps)
//   param.addcdiv_(exp_avg, denom, value = -step_size)               (a + value * (b / c))
__device__ __forceinline__ void adamw_elem(float& p, float g, float& m, float& v, float decay, const AdamWScalars& s) {
  p = __fmul_rn(p, decay);
  const float d = __fsub_rn(g, m);
  m = fabsf(s.w1) < 0.5f ? __fmaf_rn(s.w1, d, m) : __fmaf_rn(-d, __fsub_rn(1.0f, s.w1), g);
  v = __fmaf_rn(s.omb2, __fmul_rn(g, g), __fmul_rn(v, s.beta2));
  const float den = __fadd_rn(__fmul_rn(__fsqrt_rn(v), s.inv_bc2s), s.eps);
  p = __fmaf_rn(s.neg_step, __fdiv_rn(m, den), p);
}

__global__ void __launch_bounds__(kOptThreads) adamw_kernel(const __grid_constant__ OptTable t, const AdamWScalars s) {
  const int i = opt_locate(t, blockIdx.x);
  const long long lo = (long long)(blockIdx.x - t.block0[i]) * kOptChunk;
  const long long hi = min(t.n[i], lo + kOptChunk);
  float* __restrict__ P = t.p[i];
  const float* __restrict__ G = t.g[i];
  float* __restrict__ M = t.m[i];
  float* __restrict__ V = t.v[i];
  const float decay = t.decay[i];
  long long j = lo + threadIdx.x;
  if (t.vec[i]) {
    const long long hi4 = lo + ((hi - lo) & ~3ll);
#pragma unroll 2
    for (long long k = lo / 4 + threadIdx.x; k < hi4 / 4; k += kOptThreads) {
      float4 p = reinterpret_cast<float4*>(P)[k], m = reinterpret_cast<float4*>(M)[k], v = reinterpret_cast<float4*>(V)[k];
      const float4 g = __ldcs(reinterpret_cast<const float4*>(G) + k);
      adamw_elem(p.x, g.x, m.x, v.x, decay, s);
      adamw_elem(p.y, g.y, m.y, v.y, decay, s);
      adamw_elem(p.z, g.z, m.z, v.z, decay, s);
      adamw_elem(p.w, g.w, m.w, v.w, decay, s);
      reinterpret_cast<float4*>(P)[k] = p;
      reinterpret_cast<float4*>(M)[k] = m;
      reinterpret_cast<float4*>(V)[k] = v;
    }
    j = hi4 + threadIdx.x;
  }
  for (; j < hi; j += kOptThreads) {
    float p = P[j], m = M[j], v = V[j];
    adamw_elem(p, G[j], m, v, decay, s);
    P[j] = p; M[j] = m; V[j] = v;
  }
}

}  // namespace dmd
