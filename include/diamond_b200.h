/* diamond_b200 — C ABI of the GPU-native DIAMOND hot path (libdiamond_b200.so, H100 / sm_90a).
 *
 * The reference (eloialonso/diamond @ 5bcd159) is pure Python and has no FFI of its own (SURVEY.md section 8b); the
 * seam is its Python module surface.  Every entry point below therefore names the reference call site it replaces.
 * The Python mirror in diamond_b200/ binds these with ctypes (see INTEGRATION.md for the stub a maintainer adds).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host; activations are fp32
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous on it, never synchronise the device and never
 *     allocate on the hot path (the caller owns every buffer, including the workspace)
 *   - return value 0 = ok; nonzero = error, message via dmd_last_error() (thread-local)
 *   - one host thread per GPU (the reference is one process per rank, src/main.py:26)
 *
 * Workspace contract (what the caller may do with its buffers between calls; tests/test_gpu_poisoned_buffers.py checks it)
 *   Scratch -- contents undefined on entry and after the call; every byte a call reads it has written first in the same call,
 *   so the caller may reuse the memory for anything in between:
 *     - the inference workspaces of dmd_denoiser_forward, dmd_inner_model_forward[_u8], dmd_sampler_sample (also between
 *       replays of its graph), dmd_actor_critic_forward when no backward follows, dmd_rew_end_predict[_u8];
 *     - a training workspace before its *_forward_train and after its *_backward (so between optimizer steps);
 *     - the `scratch` of dmd_actor_critic_backward[_accumulate], the `partial` buffers of dmd_conv2d_wgrad, dmd_sgemm and
 *       dmd_grad_norm_clip;
 *     - every output: logits, states, model outputs, out_x, trajectory slots >= 1, the flat gradient buffer of
 *       dmd_denoiser_backward / dmd_rew_end_backward / dmd_actor_critic_backward (fully written), g_*_in, norm_coef.
 *   Kept -- must not be touched by the caller while the library relies on it:
 *     - a training workspace from dmd_inner_model_forward_train[_u8] / dmd_rew_end_forward_train[_u8] to its backward, and an
 *       actor-critic workspace from dmd_actor_critic_forward to its backward (it holds the activations);
 *     - the flat gradient buffer of dmd_actor_critic_backward_accumulate (it is added to);
 *     - the packed-weight buffers (conv packs, FiLM table and the FiLM gradient offsets, written by *_set_weights), the
 *       optimizer state (param, exp_avg, exp_avg_sq), and the frame / action rings a sampler reads (ring_head >= 0);
 *     - every input, including trajectory slot 0 and the churn noise `eps`.
 */
#ifndef DIAMOND_B200_H_
#define DIAMOND_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DMD_VERSION 101
/* Headroom of the backward loss scale: max|S * dL/d(output)| is put in [2^(E-1), 2^E), E = DMD_LOSS_SCALE_EXP, so an inner
 * gradient up to 65504 / 2^E (just under 2^(16-E)) times the largest output gradient is finite in the fp16 tensor-core operands.
 * E = 8 (headroom 256x) costs nothing measurable against E = 12 (16x) on either training fixture: fp16 keeps its relative
 * precision down to 2^-14 (oracle/grad_error_budget.py --exp emulates the scheme). */
#define DMD_LOSS_SCALE_EXP 8

int dmd_version(void);
const char* dmd_last_error(void);
/* Number of kernels launched by this library on the calling thread since the last reset (bench.py gpu_launches). */
long long dmd_launch_count(int reset);
/* Diagnostics: in-stream kernel trace.  Between dmd_ktrace_begin(capacity) and dmd_ktrace_end every conv / prep / attention /
 * wrap launch issued by this library (also into a CUDA graph being captured) gets a slot and stores the GPU nanosecond timer
 * when its inputs are ready; dmd_ktrace_end (after a device synchronisation) copies the stamps out and returns their count,
 * dmd_ktrace_name(i) describes launch i.  Differences of consecutive stamps are the in-graph kernel durations
 * (scripts/ktrace.py).  Not thread-safe; off (null slots, one predicated test per kernel) unless begun. */
int dmd_ktrace_begin(int capacity);
int dmd_ktrace_end(long long* stamps, int capacity);
const char* dmd_ktrace_name(int i);

/* ---------------------------------------------------------------------------------------------------------------
 * Per-op entry points (NHWC fp32 activations).
 * ------------------------------------------------------------------------------------------------------------- */

/* Replaces nn.Conv2d weight use (src/models/blocks.py:18-19,96): packs a torch-layout weight [Cout][CinReal][k][k]
 * into the fp16 tensor-core operand layout [taps][Cin/8][CoutPad][8].  c0_real/c0_store describe a zero-padded first
 * source (e.g. 15 real channels stored as a 16-channel operand); for an unpadded source pass c0_real = c0_store = CinReal. */
int dmd_pack_conv_weight(const float* w, void* wpk, int Cout, int CoutPad, int CinReal, int Cin, int taps,
                         int c0_real, int c0_store, int precise, void* stream);
/* precise = 1: split-fp16 packing [W_hi | W_hi | W_lo] (3*Cin channels per tap) for dmd_conv_desc.precise convs: the
 * product is evaluated as A_hi W_hi + A_lo W_hi + A_hi W_lo on the tensor cores, i.e. to ~2^-22 instead of 2^-11.  Used
 * for the layers whose input is the raw residual stream (1x1 skip projections, conv_in) and for conv_out. */

/* Activation operand ("PLC16": padded-linear, chunk-major fp16; layout in diamond_b200/csrc/conv_tc.cuh).  One pass over
 * an NHWC fp32 tensor applies what the reference runs on a conv INPUT — GroupNorm (blocks.py:28) or AdaGroupNorm
 * (blocks.py:41-45), SiLU (blocks.py:143-144), channel concat as two sources (blocks.py:174), nearest-2x upsample
 * (blocks.py:109) — and writes the operand(s) the convolution consumes. */
size_t dmd_plc16_bytes(int B, int H, int W, int C);   /* H, W: conv input size (after upsampling) */

typedef struct dmd_prep_desc {
  const float* src0;     /* NHWC [B][Hs][Ws][C0] */
  const float* src1;     /* NHWC [B][Hs][Ws][C1] or NULL */
  int C0, C1;            /* multiples of 8 */
  int B, Hs, Ws;
  int upsample;          /* 0 none ; 1 nearest-2x (blocks.py:109) ; 2 zero insertion (adjoint of the stride-2 subsample) */
  int mode;              /* 0 raw ; 1 AdaGroupNorm ; 2 affine GroupNorm */
  int silu;
  const double* stats0;  /* [B][C0/gs0][2] (sum, sumsq) */
  const double* stats1;
  int gs0, gs1;
  const float* film;     /* [B][film_stride] ; scale at film_off + c, shift at film_off + (C0+C1) + c */
  int film_stride, film_off;
  const float* gamma;    /* [C0+C1] */
  const float* beta;
  float eps;
  void* dst0;            /* operand of src0: dmd_plc16_bytes(B, H, W, C0) */
  void* dst1;
  void* dst_raw0;        /* optional: the un-normalised operand as well (1x1 skip projection, blocks.py:133,142) */
  void* dst_raw1;
  void* dst_lo0;         /* optional low parts (split-fp16): fp16(y - fp16(y)) of the transformed operand ... */
  void* dst_lo1;
  void* dst_raw_lo0;     /* ... and of the raw operand */
  void* dst_raw_lo1;
} dmd_prep_desc;

int dmd_prep_act(const dmd_prep_desc* d, void* stream);

typedef struct dmd_conv_desc {
  const void* src0;      /* PLC16 operand, C0 channels */
  const void* src1;      /* second operand (channel concat) or NULL */
  int C0, C1;            /* multiples of 16 */
  int B, H, W;           /* conv input size */
  int taps;              /* 9 = 3x3 pad 1 ; 1 = 1x1 */
  int stride;            /* 1 or 2 (blocks.py:96) */
  const void* wpk;       /* from dmd_pack_conv_weight */
  const float* bias;     /* [Cout] or NULL */
  int Cout, CoutPad;     /* CoutPad: multiple of 16, <= 128 */
  const float* residual; /* NHWC like out, or NULL (blocks.py:145) */
  float* out;            /* NHWC [B][Ho][Wo][Cout] */
  double* out_stats;     /* [B][Cout/out_gs][2], accumulated (caller zeroes) or NULL */
  int out_gs;
  int precise;           /* 1: split-fp16 (needs src*_lo and weights packed with precise = 1) */
  const void* src0_lo;
  const void* src1_lo;
  /* Optional fused 1x1 projection accumulated into the same output: out += W_x . cat(x0, x1) + b_x  (the skip path
   * r = proj(x) of ResBlock.forward, blocks.py:142,145).  Operands are split-fp16 (hi + lo), weights packed with taps = 1,
   * precise = 1. */
  const void* xsrc0; const void* xsrc1; const void* xsrc0_lo; const void* xsrc1_lo;
  int xC0, xC1;
  const void* wpk_x;
  const float* bias_x;
} dmd_conv_desc;

int dmd_conv2d_fprop(const dmd_conv_desc* d, void* stream);

/* Backward-data of nn.Conv2d = dmd_conv2d_fprop on dL/dy with the weights transposed and the taps flipped: packs
 * w'[ci][co][t'] = w[co][ci_off + ci][taps-1-t'] of a torch weight [CoutF][CinTotF][k][k] for the CinK input channels starting
 * at ci_off (one call per source of a channel concat) into [taps][round16(CoutF)/8][round16(CinK)][8] fp16. */
int dmd_pack_conv_weight_dgrad(const float* w, void* wpk, int CoutF, int CinTotF, int ci_off, int CinK, int taps, void* stream);

/* Backward-filter of nn.Conv2d (torch autograd conv2d_weight; reference forward src/models/blocks.py:18-19,96,109-110) on
 * wgmma: dW[co][ci_off+ci][t] (+)= inv_scale * sum_q GY[q][co] * X[q + o_t][ci] over the padded-linear positions of the
 * two PLC16 operands (layout and kernel: diamond_b200/csrc/wgrad_tc.cuh).  Deterministic: per-CTA partial sums are reduced in
 * a fixed order.  A stride-2 conv passes its gradient zero-inserted (dmd_prep_desc.upsample = 2) at the conv INPUT size. */
typedef struct dmd_wgrad_desc {
  const void* grad;      /* PLC16 operand of dL/dy: Cg stored channels (multiple of 8, <= 64), Cout real */
  const void* act;       /* PLC16 operand of the conv input: Ca stored channels (16 / 32 / 64), Cin real */
  int Cg, Ca;
  int B, H, W;           /* conv input size */
  int taps;              /* 9 or 1 */
  float* dW;             /* torch layout [Cout][CinTot][taps] fp32 */
  int Cout, Cin, CinTot, ci_off;
  const float* inv_scale; /* device scalar multiplied into the result, or NULL */
  int accumulate;        /* dW += instead of dW = */
  void* partial;         /* workspace of dmd_wgrad_partial_bytes() */
  size_t partial_bytes;
} dmd_wgrad_desc;
size_t dmd_wgrad_partial_bytes(void);
int dmd_conv2d_wgrad(const dmd_wgrad_desc* d, void* stream);

/* Host-only twins of dmd_conv2d_fprop / dmd_prep_act: run exactly the same validation and planning, touch neither the
 * device nor the pointed-to memory (pointers are only tested for NULL), and report the launch plan.  They make the
 * shape limits and the error behaviour (return code + dmd_last_error()) testable without a GPU. */
typedef struct dmd_conv_plan_info {
  int tiles;             /* 128-row tiles (one CTA per SM walks a contiguous range of them) */
  int kslabs;            /* 16-channel K slabs per tile, fused projection included */
  int stages;            /* depth of the shared-memory slab ring */
  int acc_cols;          /* accumulator columns of one wgmma (power of two >= CoutPad) */
  unsigned long long smem_bytes;    /* dynamic shared memory of the launch */
  unsigned long long weight_bytes;  /* resident packed weights */
} dmd_conv_plan_info;
int dmd_conv_plan(const dmd_conv_desc* d, dmd_conv_plan_info* out);
int dmd_prep_plan(const dmd_prep_desc* d, int* blocks, int* pos_per_block, int* sources);

/* GroupNorm partial sums of an NHWC tensor: stats[n][g] += (sum, sumsq) (blocks.py:28,43). */
int dmd_gn_stats(const float* x, double* stats, int B, int HW, int C, int gs, void* stream);

/* SelfAttention2d.forward (blocks.py:62-72), L = H*W = 64 tokens, C in {32, 64}, head_dim 8, groups of gs channels (gs a
 * multiple of 8 dividing C, and at L = 64 a multiple of C/4, as every model's gs = 32 is): out = xn + out_proj(softmax(q k^T
 * / sqrt(8)) v) with xn = GroupNorm(x) from the producer's statistics stats_in [B][C/gs][2]; out_stats (or NULL) [B][C/gs][2]
 * += (sum, sumsq) of out. */
int dmd_attn_fwd(const float* x, const double* stats_in, const float* gamma, const float* beta, const float* wqkv,
                 const float* bqkv, const float* wout, const float* bout, float* out, double* out_stats, int B, int L,
                 int C, int gs, float eps, void* stream);
/* dmd_attn_fwd at any token count L >= 1 (the executors' attention op).  L = 64 runs the same single launch as dmd_attn_fwd
 * and needs no scratch; any other L runs a qkv-projection kernel and a streaming-softmax kernel through `scratch`, device
 * memory of at least dmd_attn_scratch_bytes(B, L, C) bytes, 16-byte aligned. */
size_t dmd_attn_scratch_bytes(int B, int L, int C);
int dmd_attn_fwd_scratch(const float* x, const double* stats_in, const float* gamma, const float* beta, const float* wqkv,
                         const float* bqkv, const float* wout, const float* bout, float* out, double* out_stats, int B, int L,
                         int C, int gs, float eps, void* scratch, size_t scratch_bytes, void* stream);

int dmd_nchw_to_nhwc(const float* in, float* out, int B, int C, int CP, int HW, void* stream);
int dmd_nhwc_to_nchw(const float* in, float* out, int B, int C, int CP, int HW, void* stream);

/* Per-op entry points of the forward CUDA-core kernels (diamond_b200/csrc/aux_kernels.cuh) that the executors run, through
 * the same launchers, so the launch geometry is the executors'. */
/* out[n][f] (+)= silu?( sum_k in[n][k] W[f][k] + bias[f] ): the conditioning MLP (blocks.py:84-87), the batched FiLM linears
 * (blocks.py:39), the LSTM input / recurrent products and the heads (actor_critic.py:71-73, rew_end_model.py:46-55).  K a multiple
 * of 4; bias may be NULL; accumulate: out += (before the SiLU); hw_perm > 0: `in` is NHWC [B][hw_perm][K/hw_perm] read in
 * NCHW-flatten order (k = c * hw_perm + pixel, the flatten of actor_critic.py:71). */
int dmd_linear(const float* in, const float* W, const float* bias, float* out, int B, int K, int F, int silu, int accumulate,
               int hw_perm, void* stream);
/* MaxPool2d(2) (actor_critic.py:109): x NHWC [B][H][W][C] (H, W even) -> y [B][H/2][W/2][C]; stats (or NULL) [B][C/gs][2] +=
 * (sum, sumsq) of y (caller zeroes).  Statistics need gs a power of two <= 32 or a multiple of 32, and C % 32 == 0 or 256 % C == 0. */
int dmd_maxpool2_stats(const float* x, float* y, double* stats, int B, int H, int W, int C, int gs, void* stream);
/* LSTMCell pointwise part (actor_critic.py:72): gates [B][4Hd] pre-activations (order i, f, g, o), c_in [B][Hd] -> h_out, c_out
 * [B][Hd] (c_out may alias c_in). */
int dmd_lstm_gates(const float* gates, const float* c_in, float* h_out, float* c_out, int B, int Hd, void* stream);
/* Zero-pad / crop of NHWC [B][Hs][Ws][C] at the bottom / right to [B][Hd][Wd][C] (blocks.py:225-229, :245), C a multiple of 4;
 * stats (or NULL) [B][C/gs][2] += (sum, sumsq) of the result. */
int dmd_resize_nhwc(const float* src, float* dst, int B, int Hs, int Ws, int Hd, int Wd, int C, double* stats, int gs, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Per-op entry points of the CUDA-core backward kernels (diamond_b200/csrc/bwd_kernels.cuh) that dmd_denoiser_backward and
 * dmd_actor_critic_backward run, with the launch geometry those executors use.  Gradients are fp32.  `inv_scale` (a device
 * scalar, or NULL = 1) multiplies parameter gradients: the executors pass 1/S of the loss scale.
 * ------------------------------------------------------------------------------------------------------------- */

/* GroupNorm (mode 2, blocks.py:28) / AdaGroupNorm (mode 1, blocks.py:41-45) [+ SiLU] backward.  Pass 1 adds the per-(image,
 * channel) sums A = sum_px gz and Bm = sum_px gz * xhat to sumA / sumB[n * sum_stride + c] (caller zeroes them); pass 2 writes
 * gx (+ addend) or adds it to gx (accumulate).  Mode 1 reads FiLM scale at film[n * film_stride + film_off + c_off + c] and
 * shift at ... + film_ctot + c_off + c; one source of a channel concat is one launch at its channel offset c_off. */
typedef struct dmd_norm_bwd_desc {
  const float* x;        /* NHWC [B][HW][C] forward input of the norm */
  const float* gy;       /* NHWC [B][HW][C] gradient wrt the (activated) output */
  const double* stats;   /* [B][C/gs][2] forward (sum, sumsq) */
  int B, HW, C, gs;      /* C multiple of 4, <= 128; gs multiple of 4, C / gs <= 8 */
  int mode;              /* 1 AdaGroupNorm, 2 affine GroupNorm */
  int act;               /* SiLU after the norm */
  const float* film;
  int film_stride, film_off, film_ctot, c_off;
  const float* gamma;    /* mode 2: [c_off + C] */
  const float* beta;
  float eps;
  float* sumA;
  float* sumB;
  int sum_stride;
  float* gx;             /* NHWC [B][HW][C] */
  const float* addend;   /* NULL or NHWC [B][HW][C] added to gx */
  int accumulate;
} dmd_norm_bwd_desc;
int dmd_norm_bwd(const dmd_norm_bwd_desc* d, int pass, void* stream);
/* affine GroupNorm parameters after pass 1: dgamma[c] += inv_scale * sum_n sumB[n][c], dbeta[c] += inv_scale * sum_n sumA[n][c] */
int dmd_norm_affine_grad(const dmd_norm_bwd_desc* d, float* dgamma, float* dbeta, const float* inv_scale, void* stream);

/* SelfAttention2d backward (blocks.py:62-72), the forward of dmd_attn_fwd: gx (NHWC [B][L][C]) is ASSIGNED; the six parameter
 * gradients are ADDED (times inv_scale).  L = 64, C in {32, 64}. */
int dmd_attn_bwd(const float* x, const double* stats_in, const float* gamma, const float* beta, const float* wqkv, const float* bqkv,
                 const float* wout, const float* gout, float* gx, float* dgamma, float* dbeta, float* dwqkv, float* dbqkv,
                 float* dwout, float* dbout, const float* inv_scale, int B, int L, int C, int gs, float eps, void* stream);

/* C[m][n] (+)= alpha * sum_k A[m*sam + k*sak] * B[k*sbk + n*sbn] (alpha: device scalar or NULL = 1).  chunks > 1 splits K into
 * 16-aligned ranges reduced in a fixed order through `partial` (dmd_sgemm_partial_floats floats; needs ldc == N). */
long long dmd_sgemm_partial_floats(int M, int N, int K, int chunks);
int dmd_sgemm(const float* A, long long sam, long long sak, const float* B, long long sbk, long long sbn, float* C, long long ldc,
              int M, int N, int K, const float* alpha, int accumulate, int chunks, float* partial, void* stream);

/* FiLM linear weights (blocks.py:39) batched as rows of one matrix: grads[woff[f] + k] += inv_scale * sum_n dfilm[n][f] cond[n][k],
 * grads[boff[f]] += inv_scale * sum_n dfilm[n][f].  dfilm [B][rows], cond [B][CC], CC <= 256. */
int dmd_film_wgrad(const float* dfilm, const float* cond, float* grads, const long long* woff, const long long* boff, int B, int rows,
                   int CC, const float* inv_scale, void* stream);
/* act_emb (inner_model.py:27-30): dE[act[n][t]][j] += inv_scale * de[n][t * CC/T + j]; act [B][T] int64 */
int dmd_embedding_bwd(const float* de, const int64_t* act, float* dE, int B, int CC, int T, int num_actions, const float* inv_scale,
                      void* stream);
/* bias gradients: out[c] (and out2[c], if not NULL) += inv_scale * sum_rows x[row][c] for c < Creal; x [rows][C], C multiple of 4 */
int dmd_colsum(const float* x, float* out, float* out2, const float* inv_scale, long long rows, int C, int Creal, void* stream);
/* nearest-2x upsample adjoint: out [B][H][W][C] (+)= sum of the 2x2 blocks of in [B][2H][2W][C] */
int dmd_sumpool2(const float* in, float* out, int B, int H, int W, int C, int accumulate, void* stream);
/* out = dh * silu'(pre) */
int dmd_dsilu_mul(const float* pre, const float* dh, float* out, long long n, void* stream);
/* MaxPool2d(2) backward (actor_critic.py:109): y NHWC [B][H][W][C] pre-pool, gp [B][H/2][W/2][C] -> gy [B][H][W][C] (assigned) */
int dmd_maxpool2_bwd(const float* y, const float* gp, float* gy, int B, int H, int W, int C, void* stream);
/* LSTMCell backward (actor_critic.py:72): gates [B][4Hd] pre-activations, c_in [B][Hd]; g_h, g_c (either may be NULL) ->
 * dgates [B][4Hd], g_c_in [B][Hd] */
int dmd_lstm_cell_bwd(const float* gates, const float* c_in, const float* g_h, const float* g_c, float* dgates, float* g_c_in,
                      int B, int Hd, void* stream);
/* actor / critic heads (actor_critic.py:73): g_h = g_hx + g_logits Wa + g_val Wc (g_h assigned); dba += colsum(g_logits) when
 * g_logits is given; dWc += g_val^T hx_out and dbc += sum g_val when g_val is given.  Wa [A][Hd], Wc [Hd]. */
int dmd_heads_bwd(const float* g_hx, const float* g_logits, const float* g_val, const float* hx_out, const float* Wa, const float* Wc,
                  float* g_h, float* dba, float* dWc, float* dbc, int B, int Hd, int A, void* stream);
/* Loss scale of a backward call: from m = max|g| (amax: one zeroed device word), scale[0] = S (a power of two, 1 when m = 0) and
 * scale[1] = 1/S, with max|S g| in [2^(DMD_LOSS_SCALE_EXP-1), 2^DMD_LOSS_SCALE_EXP). */
int dmd_loss_scale(const float* g, long long n, unsigned int* amax, float* scale, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Denoiser executor: InnerModel.forward (inner_model.py:44-49) + Denoiser.denoise (denoiser.py:86-91) +
 * DiffusionSampler.sample (diffusion_sampler.py:31-58) as one plan of kernels, replayed as a CUDA graph.
 * ------------------------------------------------------------------------------------------------------------- */
#define DMD_MAX_LEVELS 8

typedef struct dmd_denoiser_config {
  int img_channels;             /* InnerModelConfig.img_channels */
  int num_steps_conditioning;   /* frame stack */
  int cond_channels;
  int num_levels;
  int depths[DMD_MAX_LEVELS];
  int channels[DMD_MAX_LEVELS];
  int attn_depths[DMD_MAX_LEVELS];
  int num_actions;
  float sigma_data;             /* DenoiserConfig */
  float sigma_offset_noise;
} dmd_denoiser_config;

typedef struct dmd_denoiser dmd_denoiser;

/* Frames stored as one byte per value (Episode.save's levels, src/data/episode.py:47), read in place through strides.
 * Frame (n, f) of the source -- sample n, frame f -- is C*H*W contiguous bytes at levels + n * batch_stride + f * frame_stride
 * (strides in bytes), and has one kind byte at kinds[n * kind_batch_stride + f * kind_frame_stride].  Value i of the frame is
 * table[kind * 256 + byte]: table (DMD_FRAME_KINDS x 256 fp32, device memory) holds, per kind, the value the fp32 entry point
 * would have read for that byte, so the two entry points compute the same thing (diamond_b200/frames.py builds the tables).
 * Kinds: 0 padding (0.0 whatever the byte), 1 decoded on the CPU (Episode.load, src/data/episode.py:39), 2 decoded on the
 * GPU by torch (the denoiser's quantiser write-back, a real env's final observation).  A kind >= DMD_FRAME_KINDS reads as 0.
 * A (B, T, C, H, W) uint8 tensor with its (B, T) kinds gives frames [i, i + n) as levels + i * C*H*W, kinds + i. */
#define DMD_FRAME_KINDS 3
typedef struct dmd_u8_frames {
  const uint8_t* levels;
  long long batch_stride;
  long long frame_stride;
  const uint8_t* kinds;
  long long kind_batch_stride;
  long long kind_frame_stride;
  const float* table;
} dmd_u8_frames;

dmd_denoiser* dmd_denoiser_create(const dmd_denoiser_config* cfg);
void dmd_denoiser_destroy(dmd_denoiser* h);

/* Number of parameter/buffer tensors expected by dmd_denoiser_set_weights == len(InnerModel.state_dict()). */
int dmd_denoiser_num_tensors(const dmd_denoiser* h);
/* Bytes of device memory needed for packed weights (caller allocates, passes to set_weights). */
size_t dmd_denoiser_packed_bytes(const dmd_denoiser* h);
/* ptrs_host: host array of device pointers, in InnerModel.state_dict() order (fp32, torch layouts).
 * Re-packs the tensor-core copies; call again after every optimizer step / load_state_dict. */
int dmd_denoiser_set_weights(dmd_denoiser* h, const float* const* ptrs_host, int n_ptrs, void* packed, void* stream);

/* H, W need not be multiples of 2^(levels-1): like UNet.forward (blocks.py:225-229,245) the executor zero-pads the conv_in
 * output at the bottom / right, runs the U-Net on the padded size and crops before norm_out / conv_out (inference entry
 * points; the training entry points reject such sizes).  Attention runs over any token count at inference, and the workspace
 * includes its scratch; the training entry points reject an attention block over other than 8x8 = 64 positions (the attention
 * backward is built for 64 tokens only) before any launch. */
size_t dmd_denoiser_workspace_bytes(const dmd_denoiser* h, int B, int H, int W);

/* One Denoiser.denoise / compute_model_output call.  noisy (B,C,H,W), sigma (B) or (1), obs (B,T*C,H,W),
 * act (B,T) int64.  out_model / out_denoised are NCHW (B,C,H,W); either may be NULL. */
int dmd_denoiser_forward(dmd_denoiser* h, int B, int H, int W, const float* noisy, const float* sigma,
                         int sigma_is_scalar, const float* obs, const int64_t* act, float* out_model,
                         float* out_denoised, void* workspace, size_t workspace_bytes, void* stream);

/* InnerModel.forward (inner_model.py:44-49): inputs already rescaled by the caller (denoiser.py:75-76), c_noise (B) or
 * (1).  out: (B,C,H,W) NCHW model output. */
int dmd_inner_model_forward(dmd_denoiser* h, int B, int H, int W, const float* noisy_rescaled, const float* c_noise,
                            int c_noise_is_scalar, const float* obs_rescaled, const int64_t* act, float* out,
                            void* workspace, size_t workspace_bytes, void* stream);

/* ---- Training (Denoiser.forward + loss.backward(), src/models/diffusion/denoiser.py:93-122, src/trainer.py:365-366).
 * dmd_inner_model_forward_train = dmd_inner_model_forward that keeps every activation (and the GroupNorm statistics) in the
 * training workspace; dmd_denoiser_backward consumes them: given dL/d(model output) (B,C,H,W) it writes the gradient of
 * EVERY parameter into one flat fp32 buffer (16-byte aligned slices, layout from dmd_denoiser_grad_layout, state_dict
 * order; buffers such as noise_emb.weight get zeros).  Convolutions run on wgmma (dgrad = fprop with transposed weights,
 * wgrad = dmd_conv2d_wgrad), gradients carry a power-of-two loss scale chosen from max|grad_out| on the device.  The flat
 * buffer is what a data-parallel step all-reduces in ONE collective (utils.py:105-106 wraps each model in DDP instead). */
size_t dmd_denoiser_train_workspace_bytes(const dmd_denoiser* h, int B, int H, int W);
/* offsets / numels: n = dmd_denoiser_num_tensors entries (floats); returns the total length of the flat buffer. */
long long dmd_denoiser_grad_layout(const dmd_denoiser* h, long long* offsets, long long* numels, int n);
int dmd_inner_model_forward_train(dmd_denoiser* h, int B, int H, int W, const float* noisy_rescaled, const float* c_noise,
                                  int c_noise_is_scalar, const float* obs_rescaled, const int64_t* act, float* out,
                                  void* workspace, size_t workspace_bytes, void* stream);
int dmd_denoiser_backward(dmd_denoiser* h, int B, int H, int W, const float* grad_out, float* grads, long long grads_numel,
                          void* workspace, void* stream);

/* dmd_inner_model_forward / dmd_inner_model_forward_train with the frame stack read from uint8 frames: obs holds the
 * num_steps_conditioning frames of each sample, f = 0 oldest, and its table the rescaled values obs / sigma_data (what
 * obs_rescaled would hold).  dmd_denoiser_backward is the same after either forward.  Every argument is checked before
 * any launch. */
int dmd_inner_model_forward_u8(dmd_denoiser* h, int B, int H, int W, const float* noisy_rescaled, const float* c_noise,
                               int c_noise_is_scalar, const dmd_u8_frames* obs, const int64_t* act, float* out,
                               void* workspace, size_t workspace_bytes, void* stream);
int dmd_inner_model_forward_train_u8(dmd_denoiser* h, int B, int H, int W, const float* noisy_rescaled, const float* c_noise,
                                     int c_noise_is_scalar, const dmd_u8_frames* obs, const int64_t* act, float* out,
                                     void* workspace, size_t workspace_bytes, void* stream);

typedef struct dmd_sampler_config {
  int num_sigmas;               /* len(self.sigmas) = num_steps_denoising + 1, last one 0 */
  const float* sigmas_host;     /* host array, fp32 values of DiffusionSampler.sigmas */
  int order;                    /* 1 Euler, 2 Heun */
  float s_churn, s_tmin, s_tmax, s_noise;
} dmd_sampler_config;

/* DiffusionSampler.sample (src/models/diffusion/diffusion_sampler.py:31-58), whole loop in one call, replayed as a CUDA graph.
 * Every buffer is used IN PLACE (no staging copies; a graph is cached per distinct set of addresses):
 *   traj  (num_sigmas, B, C, H, W): slot 0 holds the initial x ~ N(0,1) on entry (drawn by the CALLER with torch so that RNG
 *         streams match the reference, :36); slot i+1 receives the iterate after step i (the reference's `trajectory`).
 *   eps   (num_steps, B, C, H, W) churn noise (:42) or NULL.
 *   out_x (B, C, H, W) or NULL: additionally receives the final iterate (e.g. a slot of the caller's frame ring).
 *   ring_head = -1: prev_obs (B, T*C, H, W), prev_act (B, T) as the reference passes them.
 *   ring_head >= 0: the WorldModelEnv's resident buffers -- prev_obs = frames (T, B, C, H, W), prev_act = actions (T, B), where
 *         LOGICAL slot k (0 = oldest) is physical slot (ring_head + k) % T: the per-step `roll` of both buffers
 *         (src/envs/world_model_env.py:74-75) becomes an index increment.
 * The conditioning path (Fourier + action embedding -> MLP -> all FiLM linears) of all denoising steps is evaluated once, up
 * front: the sigma schedule is host-known (:27) and the actions are fixed during a call. */
int dmd_sampler_sample(dmd_denoiser* h, const dmd_sampler_config* sc, int B, int H, int W, const float* prev_obs,
                       const int64_t* prev_act, int ring_head, float* traj, const float* eps, float* out_x, void* workspace,
                       size_t workspace_bytes, int use_graph, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Actor-critic executor: ActorCritic.predict_act_value (src/models/actor_critic.py:68-73) = ActorCriticEncoder
 * (:101-113: Conv3x3 + [SmallResBlock (blocks.py:116-123), MaxPool2d]*) -> flatten -> LSTMCell -> actor / critic heads.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct dmd_actor_critic_config {
  int lstm_dim;
  int img_channels;
  int img_size;
  int num_levels;
  int channels[DMD_MAX_LEVELS];
  int down[DMD_MAX_LEVELS];
  int num_actions;
} dmd_actor_critic_config;

typedef struct dmd_actor_critic dmd_actor_critic;

dmd_actor_critic* dmd_actor_critic_create(const dmd_actor_critic_config* cfg);
void dmd_actor_critic_destroy(dmd_actor_critic* h);
int dmd_actor_critic_num_tensors(const dmd_actor_critic* h);          /* == len(ActorCritic.state_dict()) */
size_t dmd_actor_critic_packed_bytes(const dmd_actor_critic* h);
int dmd_actor_critic_set_weights(dmd_actor_critic* h, const float* const* ptrs_host, int n_ptrs, void* packed, void* stream);
size_t dmd_actor_critic_workspace_bytes(const dmd_actor_critic* h, int B);
/* obs (B,C,S,S) NCHW; hx_in/cx_in (B,lstm_dim); outputs: logits (B,A), val (B), hx_out/cx_out (B,lstm_dim). */
int dmd_actor_critic_forward(dmd_actor_critic* h, int B, const float* obs, const float* hx_in, const float* cx_in,
                             float* logits, float* val, float* hx_out, float* cx_out, void* workspace,
                             size_t workspace_bytes, void* stream);

/* ---- Actor-critic training: ActorCritic.predict_act_value under autograd (src/models/actor_critic.py:68-73; the imagined
 * rollout calls it with grad, src/coroutines/env_loop.py:31,57, and src/trainer.py:366 back-propagates through time).
 * dmd_actor_critic_forward leaves every activation in its workspace; ONE dmd_actor_critic_backward call is one node of the
 * BPTT graph: given the gradients wrt (logits, val, hx_out, cx_out) (any may be NULL = zero) it writes the gradients wrt
 * (hx_in, cx_in) and the gradient of every parameter into a flat fp32 buffer (layout: dmd_actor_critic_grad_layout).
 * `workspace` is the forward's (untouched since); `scratch` is transient and may be shared by all nodes of a stream. */
size_t dmd_actor_critic_backward_scratch_bytes(const dmd_actor_critic* h, int B);
long long dmd_actor_critic_grad_layout(const dmd_actor_critic* h, long long* offsets, long long* numels, int n);
int dmd_actor_critic_backward(dmd_actor_critic* h, int B, const float* hx_in, const float* cx_in, const float* hx_out,
                              const float* g_logits, const float* g_val, const float* g_hx, const float* g_cx, float* grads,
                              long long grads_numel, float* g_hx_in, float* g_cx_in, void* workspace, void* scratch,
                              size_t scratch_bytes, void* stream);
/* Same, but ADDS the parameter gradients to what `grads` already holds: the nodes of one back-propagation-through-time pass
 * accumulate into one flat buffer (what autograd's AccumulateGrad does tensor by tensor in the reference, trainer.py:366). */
int dmd_actor_critic_backward_accumulate(dmd_actor_critic* h, int B, const float* hx_in, const float* cx_in, const float* hx_out,
                                         const float* g_logits, const float* g_val, const float* g_hx, const float* g_cx,
                                         float* grads, long long grads_numel, float* g_hx_in, float* g_cx_in, void* workspace,
                                         void* scratch, size_t scratch_bytes, void* stream);

/* compute_lambda_returns (src/models/actor_critic.py:116-143): rew / val_bootstrap fp32 [B][T], end / trunc int64 [B][T] ->
 * out fp32 [B][T]; one thread per environment walks time backwards; bit-identical to the reference's torch expression. */
int dmd_lambda_returns(const float* rew, const int64_t* end, const int64_t* trunc, const float* val_bootstrap, float* out, int B,
                       int T, double gamma, double lambda_, void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Reward / termination model: RewEndModel.predict_rew_end (src/models/rew_end_model.py:42-55; SURVEY.md 8 f1), called once
 * per imagined step (src/envs/world_model_env.py:97) and over the burn-in frames of each fresh episode (:120-129).
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct dmd_rew_end_config {
  int lstm_dim;
  int img_channels;
  int img_size;
  int cond_channels;
  int num_levels;
  int depths[DMD_MAX_LEVELS];
  int channels[DMD_MAX_LEVELS];
  int attn_depths[DMD_MAX_LEVELS];
  int num_actions;
} dmd_rew_end_config;
typedef struct dmd_rew_end dmd_rew_end;
dmd_rew_end* dmd_rew_end_create(const dmd_rew_end_config* cfg);
void dmd_rew_end_destroy(dmd_rew_end* h);
int dmd_rew_end_num_tensors(const dmd_rew_end* h);           /* == len(RewEndModel.state_dict()) */
size_t dmd_rew_end_packed_bytes(const dmd_rew_end* h);
int dmd_rew_end_set_weights(dmd_rew_end* h, const float* const* ptrs_host, int n_ptrs, void* packed, void* stream);
size_t dmd_rew_end_workspace_bytes(const dmd_rew_end* h, int rows);  /* rows = b * t */
/* obs / next_obs (b, t, C, S, S), act (b, t) int64, hx_in / cx_in (b, lstm_dim) or NULL (zero state).
 * logits_rew (b, t, 3), logits_end (b, t, 2), hx_out / cx_out (b, lstm_dim). */
int dmd_rew_end_predict(dmd_rew_end* h, int b, int t, const float* obs, const float* next_obs, const int64_t* act,
                        const float* hx_in, const float* cx_in, float* logits_rew, float* logits_end, float* hx_out,
                        float* cx_out, void* workspace, size_t workspace_bytes, void* stream);

/* ---- Reward / termination training: RewEndModel.predict_rew_end under autograd (RewEndModel.forward,
 * src/models/rew_end_model.py:57-90).  dmd_rew_end_forward_train = dmd_rew_end_predict that keeps every activation (encoder,
 * the gates and states of every LSTM step, the head's hidden layer) in the training workspace of (b, t);
 * dmd_rew_end_backward consumes them: given the gradients wrt (logits_rew, logits_end) and optionally (hx_out, cx_out)
 * (NULL = zero) it writes the gradient of EVERY parameter into one flat fp32 buffer (layout: dmd_rew_end_grad_layout,
 * state_dict order, fully written) and, when the pointers are not NULL, the gradients wrt (hx_in, cx_in).  The LSTM and head
 * gradients are fp32; the encoder's run on the same wgmma backward as the denoiser's, under a power-of-two loss scale. */
size_t dmd_rew_end_train_workspace_bytes(const dmd_rew_end* h, int b, int t);
long long dmd_rew_end_grad_layout(const dmd_rew_end* h, long long* offsets, long long* numels, int n);
int dmd_rew_end_forward_train(dmd_rew_end* h, int b, int t, const float* obs, const float* next_obs, const int64_t* act,
                              const float* hx_in, const float* cx_in, float* logits_rew, float* logits_end, float* hx_out,
                              float* cx_out, void* workspace, size_t workspace_bytes, void* stream);
int dmd_rew_end_backward(dmd_rew_end* h, int b, int t, const float* g_logits_rew, const float* g_logits_end,
                         const float* g_hx_out, const float* g_cx_out, float* grads, long long grads_numel,
                         float* g_hx_in, float* g_cx_in, void* workspace, void* stream);
/* dmd_rew_end_predict / dmd_rew_end_forward_train with obs / next_obs read from uint8 frames (frame (n, k) = step k of
 * segment n); both sources share one decode table (values as the fp32 entry points read them).  dmd_rew_end_backward is the
 * same after either forward.  Every argument is checked before any launch. */
int dmd_rew_end_predict_u8(dmd_rew_end* h, int b, int t, const dmd_u8_frames* obs, const dmd_u8_frames* next_obs,
                           const int64_t* act, const float* hx_in, const float* cx_in, float* logits_rew, float* logits_end,
                           float* hx_out, float* cx_out, void* workspace, size_t workspace_bytes, void* stream);
int dmd_rew_end_forward_train_u8(dmd_rew_end* h, int b, int t, const dmd_u8_frames* obs, const dmd_u8_frames* next_obs,
                                 const int64_t* act, const float* hx_in, const float* cx_in, float* logits_rew,
                                 float* logits_end, float* hx_out, float* cx_out, void* workspace, size_t workspace_bytes,
                                 void* stream);

/* ---------------------------------------------------------------------------------------------------------------
 * Optimizer: torch.nn.utils.clip_grad_norm_ + torch.optim.AdamW (src/trainer.py:373-377, src/utils.py:164) over every
 * tensor of a parameter list, one launch per kernel for up to 512 non-empty tensors (diamond_b200/optim.py).  The table is
 * HOST memory, read at call time; every pointer in it is a device pointer to contiguous fp32 data.  Arguments are checked
 * before any CUDA call.
 * ------------------------------------------------------------------------------------------------------------- */
typedef struct dmd_optim_tensor {
  float* param;          /* AdamW only */
  float* grad;
  float* exp_avg;        /* AdamW only */
  float* exp_avg_sq;     /* AdamW only */
  long long numel;       /* >= 0; 0 = skipped */
  double weight_decay;   /* AdamW only: the tensor's group value */
} dmd_optim_tensor;
/* Bytes of the fp64 per-block partial buffer dmd_grad_norm_clip needs for this table (0 on an invalid table). */
size_t dmd_grad_norm_partial_bytes(const dmd_optim_tensor* table_host, int n);
/* Squared 2-norm in fp64 per block, reduced in a fixed order (repeat runs are bit-identical); then norm_coef[0] = total_norm
 * (fp32) and norm_coef[1] = min(1, max_norm / (total_norm + 1e-6)) computed as torch does (a NaN norm gives a NaN coefficient);
 * with clip != 0 every grad is then multiplied by norm_coef[1] in place (not read or written when it is exactly 1).  No host
 * synchronisation.  3 launches (norm, reduction, scale); clip = 0 leaves out the scale. */
int dmd_grad_norm_clip(const dmd_optim_tensor* table_host, int n, double max_norm, int clip, float* norm_coef, void* partial,
                       size_t partial_bytes, void* stream);
/* One AdamW step of torch 2.11 (decoupled weight decay, amsgrad / maximize off) at step count `step` (>= 1, after the
 * increment) for every tensor of the table; lr, betas, eps are the group's, weight decay the table entry's. */
int dmd_adamw_step(const dmd_optim_tensor* table_host, int n, double lr, double beta1, double beta2, double eps, double step,
                   void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIAMOND_B200_H_ */
