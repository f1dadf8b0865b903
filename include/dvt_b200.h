/*
 * dvt_b200 -- C ABI of the H100-native (sm_90a) hot paths of Denoising-ViT (DVT).
 *
 * The reference (Jiawei-Yang/Denoising-ViT) has no FFI layer of its own: its hot paths are reached through the
 * Python API of `dvt.models`, which in turn calls timm (ViT forward), tiny-cuda-nn (hash-grid encoding) and
 * torch (Linear / grid_sample / Adam).  This header is the boundary a maintainer binds instead of those
 * libraries; every entry point cites the reference interface it replaces.  See INTEGRATION.md for the ctypes
 * stubs on the reference side.
 *
 * Conventions
 *   - every function returns 0 on success; non-zero codes are DVT_ERR_*; dvt_last_error() gives the message
 *     (thread-local).  Nothing aborts the process.
 *   - all tensor pointers are DEVICE pointers owned by the caller unless a parameter name ends in `_host`.
 *   - `stream` is a cudaStream_t passed as void*; work is enqueued, not synchronised.
 *   - hot calls do not allocate: handles own their workspaces, sized at create time.
 *   - bf16 tensors are passed as void* (uint16 storage).
 */
#ifndef DVT_B200_H_
#define DVT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DVT_OK 0
#define DVT_ERR_INVALID 1
#define DVT_ERR_CUDA 2
#define DVT_ERR_DEVICE 3

#define DVT_DTYPE_BF16 0
#define DVT_DTYPE_F32 1

/* ---------------------------------------------------------------------------------------------------------
 * library
 * ------------------------------------------------------------------------------------------------------- */
int dvt_version(void);
const char* dvt_last_error(void);
/* Reads (and clears) the device-side error word written by a kernel watchdog; 0 = none. */
int dvt_device_error(unsigned int* code_out);
/* Number of kernels this library has launched in the calling process (CUDA-graph replays count their nodes). */
long long dvt_launch_count(void);
/* Process-wide kernel implementation switch for debugging, for every GEMM and the attention forward without lse:
 * 0 = tensor-core kernels (wgmma / mma.sync; default), 1 = plain SIMT reference kernels (same semantics, slow; also
 * settable with DVT_GEMM_IMPL=simt), -1 = back to the DVT_GEMM_IMPL default.  Read when a call enqueues its kernels
 * (for dvt_fit_run with graphs: when the graph is captured). */
int dvt_set_debug_impl(int impl);

/* ---------------------------------------------------------------------------------------------------------
 * unit operators (kernel-level parity tests; each is also a building block of the two paths below)
 * ------------------------------------------------------------------------------------------------------- */

/* C[M,N] = act(A[M,K] . B[N,K]^T + bias) with A, B row-major, K contiguous (torch nn.Linear convention:
 * B is the Linear weight).  dtype: DVT_DTYPE_BF16 (bf16 operands) or DVT_DTYPE_F32 (fp32 operands, TF32
 * tensor-core math).  act: 0 none, 1 GELU(erf), 2 ReLU.  out_dtype: bf16 or f32.  splits > 1 accumulates
 * split-K partial sums atomically into a zero-initialised fp32 `out` (no bias, no activation).  The epilogue accesses
 * four columns at once: `out` must be 16-byte aligned (f32) or 8-byte aligned (bf16), `bias` 16-byte aligned, ldo a
 * multiple of 4; A and B 16-byte aligned with row pitches that are multiples of 16 bytes.  GELU(NaN) = NaN.
 * Replaces: torch.nn.Linear / cuBLAS calls made by timm Block (qkv, proj, fc1, fc2) and by
 * dvt/models/neural_feature_field.py:40-44, dvt/models/offline_denoiser.py:40-46. */
int dvt_gemm_tn(const void* A, int lda, const void* B, int ldb, int dtype, int M, int N, int K, const float* bias,
                int act, void* out, int ldo, int out_dtype, int splits, void* stream);

/* out[m,n] += gamma[n] * (A.B^T + bias)[m,n] on an fp32 residual stream (LayerScale + residual add; gamma NULL: unit
 * scale).  branch_out_bf16 (optional, [M, ld_branch], ld_branch >= N and a multiple of 4): also writes the pre-LayerScale
 * branch value A.B^T + bias as bf16 (what dvt_layerscale_bwd needs); x_inout is updated identically with or without it.
 * Alignment: x_inout, bias and gamma 16 bytes, branch_out_bf16 8 bytes (as for dvt_gemm_tn).
 * Replaces: `x = x + ls(attn(...))` / `x = x + ls(mlp(...))` in timm Block.forward
 * (restated in the reference at evaluation/vitdet/vision_transformer.py:98-117). */
int dvt_gemm_tn_residual(const void* A, int lda, const void* B, int ldb, int dtype, int M, int N, int K,
                         const float* bias, const float* gamma, float* x_inout, int ldx, void* branch_out_bf16,
                         int ld_branch, void* stream);

/* y = LayerNorm(x) over rows of C fp32 (eps inside the sqrt, affine gamma/beta), output bf16 or fp32.
 * in_group/skip: rows are grouped in runs of `in_group`; the first `skip` rows of every group are dropped and the
 * output is compacted (used to strip prefix tokens); pass in_group=1, skip=0 for a plain LayerNorm.  0 <= skip < in_group,
 * and rows % in_group == 0 when skip > 0.  C % 4 == 0, 4 <= C <= 2048; ldx, ldy >= C and multiples of 4.  Alignment:
 * x, gamma and beta 16 bytes; y 16 bytes (f32) or 8 bytes (bf16).
 * Replaces: nn.LayerNorm(eps=1e-6) in timm Block / VisionTransformer.norm. */
int dvt_layernorm(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int y_dtype,
                  int rows, int C, float eps, int in_group, int skip, void* stream);

/* Multi-head attention, no mask, head_dim 64 or 80 (80: ViT-H/14), scale head_dim^-0.5: qkv bf16 [B, N, 3*heads*head_dim]
 * -> out bf16 [B, N, heads*head_dim].  lse (optional, for the backward): f32 [B, heads, N], the log2-domain log-sum-exp of
 * the scaled scores; a call with lse always runs the tensor-core kernel (the SIMT debug kernel has no lse output), one
 * without follows dvt_set_debug_impl.  out is the same with or without lse.
 * Replaces: timm Attention.forward -> F.scaled_dot_product_attention
 * (reference restatement: evaluation/vitdet/vision_transformer.py:73-91). */
int dvt_attention_fwd(const void* qkv_bf16, void* out_bf16, float* lse, int B, int N, int heads, int head_dim,
                      void* stream);

/* Patch extraction for Conv2d(3->C, kernel P, stride S): x [B,3,H,W] (f32 or bf16) -> bf16 [B*h*w, Kp],
 * Kp = round_up(3*P*P, 8), column = c*P*P + i*P + j.  h = (H-P)/S+1, w = (W-P)/S+1
 * (dvt/models/vit_wrapper.py:78-91: stride override + dynamic_feat_size). */
int dvt_im2col(const void* x, int x_dtype, void* out_bf16, int B, int H, int W, int P, int S, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * HP-1: frozen ViT forward (replaces PretrainedViTWrapper.get_intermediate_layers,
 * dvt/models/vit_wrapper.py:122-143, i.e. timm VisionTransformer.forward_intermediates)
 * ------------------------------------------------------------------------------------------------------- */
typedef struct dvt_vit dvt_vit_t;

/* prefix_tokens = 1 (cls) + number of register tokens.  head_dim = embed / heads is 64 or 80.  pre_norm != 0: a
 * LayerNorm `norm_pre` (weights loaded as "norm_pre.weight" / "norm_pre.bias") over all token rows between the token
 * assembly and the first block (timm pre_norm=True: the CLIP towers).  patch_bias == 0: the patch embedding has no bias
 * ("patch_embed.proj.bias" is not a key).  ln_eps applies to every LayerNorm.  rope != 0: 2-D rotary position embedding
 * (DINOv3; head_dim 64) on q and k of the patch tokens, fused into the epilogue of the QKV GEMM, and no absolute position
 * term (dvt_vit_forward takes the RoPE table instead of pos_patch). */
int dvt_vit_create(dvt_vit_t** out, int embed, int depth, int heads, int patch, int mlp_hidden, int swiglu,
                   int layerscale, int prefix_tokens, float ln_eps, int pre_norm, int patch_bias, int rope);
void dvt_vit_destroy(dvt_vit_t* h);
/* Loads one fp32 tensor by its timm state-dict key (without the wrapper's "model." prefix), e.g.
 * "blocks.3.attn.qkv.weight".  `src` may be host or device memory.  cls_token / reg_token / pos_embed are not
 * loaded here: the caller passes the (resampled) position table and the prefix rows to dvt_vit_forward. */
int dvt_vit_load(dvt_vit_t* h, const char* timm_key, const float* src, size_t numel);
/* Pre-sizes the activation workspaces (otherwise grown on first use). */
int dvt_vit_reserve(dvt_vit_t* h, int max_batch, int H, int W, int stride);
/* x: [B,3,H,W] f32 or bf16.  pos_patch: f32 [h*w, C] position embedding of the patch tokens for this grid
 * (already resampled; NULL for a RoPE ViT).  prefix_rows: f32 [prefix_tokens, C] rows written in front of the patches
 * (cls + its position, register tokens).  rope (RoPE ViTs only, else NULL): f32 [h*w, 64], row p = (cos | sin) of the 32
 * angles of patch p (dvt_gemm_qkv_rope).  16-byte aligned tables.  Runs blocks 0..layer_index, applies the final
 * LayerNorm if `norm`.  out (f32): all_tokens == 0 -> [B, h, w, C] (prefix stripped, NHWC); all_tokens == 1 ->
 * [B, prefix + h*w, C]. */
int dvt_vit_forward(dvt_vit_t* h, const void* x, int x_dtype, int B, int H, int W, int stride,
                    const float* pos_patch, const float* prefix_rows, const float* rope, int layer_index, int norm,
                    float* out, int all_tokens, void* stream);
/* dvt_vit_forward for several layers in one pass: runs blocks 0..layer_indices[n_layers-1] once and, after block
 * layer_indices[l], writes the map of that layer (final LayerNorm if `norm`, as dvt_vit_forward) into out[l] at row pitch
 * `ldo` floats (ldo >= C, a multiple of 4; out[l] 16-byte aligned): all_tokens == 0 -> [B, h, w, C] rows, all_tokens == 1
 * -> [B, prefix + h*w, C] rows.  layer_indices (host array) is strictly ascending within [0, depth); out and prefix_out
 * are host arrays of n_layers device pointers.  With ldo = n_layers*C and out[l] = base + l*C the maps land
 * channel-concatenated, [B, h, w, n_layers*C].  prefix_out (optional, not with all_tokens): prefix_out[l] receives the
 * prefix rows of layer l, [B, prefix_tokens, C] at pitch C, normalised like out[l].  Each map has the bits dvt_vit_forward
 * gives for that layer. */
int dvt_vit_forward_layers(dvt_vit_t* h, const void* x, int x_dtype, int B, int H, int W, int stride,
                           const float* pos_patch, const float* prefix_rows, const float* rope, int n_layers,
                           const int* layer_indices, int norm, float* const* out, int ldo, int all_tokens,
                           float* const* prefix_out, void* stream);

/* General form of dvt_gemm_tn for bf16 operands, no bias or activation: a_mn / b_mn = 1 reads the operand from its
 * transposed storage ([K, M] / [K, N] row-major, "MN-major") without a copy.  Supported: (a_mn, b_mn) in {(0,0), (0,1),
 * (1,1)}.  Used for the backward GEMMs: data gradients (b_mn = 1: the weight is read in its [out, in] storage) and weight
 * gradients (a_mn = b_mn = 1: activations read in their [rows, features] storage, split-K over the rows).
 *   splits > 1: partial sums added with f32 atomics into a zero-initialised `out`.
 *   gelu_preact_bf16 (optional, [M, ld_preact], 8-byte aligned, ld_preact a multiple of 4): the GELU derivative fused
 *     into the epilogue, out = (A.B^T) * gelu'(gelu_preact[m, n]) (replaces autograd through nn.GELU).
 *   last_col_out (optional): column N-1 of the product is accumulated into last_col_out[M] instead of out (bias gradient
 *     via a ones column in B).
 * splits > 1 and last_col_out accumulate, so they need out_dtype f32 and no gelu_preact. */
int dvt_gemm_bf16(const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, int M, int N, int K, void* out,
                  int ldo, int out_dtype, int splits, const void* gelu_preact_bf16, int ld_preact, float* last_col_out,
                  void* stream);

/* fp32-accurate GEMM on the tensor cores ("3xTF32"): every fp32 operand is given as two planes, hi = the TF32-exact
 * part (low 13 mantissa bits zero) at the pointer and lo = x - hi at pointer + plane (elements); the kernel
 * accumulates A_hi.B_hi + A_hi.B_lo + A_lo.B_hi in fp32.  a_mn / b_mn as in dvt_gemm_bf16.  This is what the
 * stage-1 fit uses for nn.Linear forward/backward (the reference runs them in fp32 on cuBLAS:
 * dvt/models/neural_feature_field.py:40-44, dvt/models/offline_denoiser.py:40-46 with --dtype float32). */
int dvt_gemm_f32x3(const float* A, int lda, size_t plane_a, int a_mn, const float* B, int ldb, size_t plane_b, int b_mn,
                   int M, int N, int K, float* out, int ldo, int splits, float* last_col_out, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * multiresolution hash grid, 2-D inputs, 8 features per level (replaces tcnn.Encoding(HashGrid) created at
 * dvt/models/neural_feature_field.py:25-39).  The level table (scale, resolution, entries, offsets, hashed flag per
 * level) is computed by the caller exactly as tiny-cuda-nn does (dvt/models/hashgrid_meta.py) and passed in:
 * HOST arrays scale[L] (f32), res[L], size[L], offset[L+1], hashed[L] (u32).
 * ------------------------------------------------------------------------------------------------------- */
/* idx [n, L, 4] u32 (entry index incl. level offset) and w [n, L, 4] f32 of the 4 interpolation corners. */
int dvt_hashgrid_corners(int n_levels, const float* scale_host, const uint32_t* res_host, const uint32_t* size_host,
                         const uint32_t* offset_host, const uint32_t* hashed_host, const float* coords, int n,
                         uint32_t* idx_out, float* w_out, void* stream);
/* out [n, L*8] f32 = encoding of coords [n, 2] with table [entries, 8] f32. */
int dvt_hashgrid_fwd(int n_levels, const float* scale_host, const uint32_t* res_host, const uint32_t* size_host,
                     const uint32_t* offset_host, const uint32_t* hashed_host, const float* table, const float* coords,
                     int n, float* out, void* stream);
/* grad_table [entries, 8] f32 += d out / d table contracted with dout [n, L*8] (dense gradient, like tcnn). */
int dvt_hashgrid_bwd(int n_levels, const float* scale_host, const uint32_t* res_host, const uint32_t* size_host,
                     const uint32_t* offset_host, const uint32_t* hashed_host, const float* coords, int n,
                     const float* dout, float* grad_table, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * HP-2: per-image neural-field fit (replaces the loop of denoise_an_image, main_img_denoising.py:39-89, i.e.
 * SingleImageDenoiser.forward + NeuralFeatureField.forward + torch.optim.Adam.step per iteration)
 * ------------------------------------------------------------------------------------------------------- */
typedef struct dvt_fit dvt_fit_t;

/* feat_dim C (multiple of 32), noise map gh x gw, pixel batch `bsz` (args.pixel_bsz), hash-grid level table. */
int dvt_fit_create(dvt_fit_t** out, int feat_dim, int gh, int gw, int bsz, int n_levels, const float* scale_host,
                   const uint32_t* res_host, const uint32_t* size_host, const uint32_t* offset_host,
                   const uint32_t* hashed_host);
void dvt_fit_destroy(dvt_fit_t* h);
/* Stream discipline: calls that change engine state (init_params, set_param, begin, run) are ordered after the work
 * already enqueued on `stream` and run on the engine's own streams; calls that read state (query, residual,
 * losses_async) are ordered after the engine on `stream`.  None of them waits for the device on the host unless stated,
 * so a driver can enqueue the next image while the current fit is running. */
/* Parameters by name, fp32, host or device: "G" (shared_artifacts [1,C,gh,gw]), "res.{0,2,4}.{weight,bias}"
 * (residual_predictor), "table" (tcnn params, [entries*8]), "mlp.{0,2}.{weight,bias}" (NeuralFeatureField.mlp). */
int dvt_fit_set_param(dvt_fit_t* h, const char* name, const float* src, size_t numel, void* stream);
/* dvt_fit_get_param also reads the optimiser state: "<name>.m" / "<name>.v" are the Adam moments of any of the names
 * above, in the parameter's own layout ("G.m" / "G.v" as [1,C,gh,gw]); "table.next" is the table buffer the next sweep
 * writes. */
int dvt_fit_get_param(dvt_fit_t* h, const char* name, float* dst, size_t numel);   /* blocks */
/* Fresh parameters for the next fit, drawn on the device from a counter-based generator: what constructing new
 * SingleImageDenoiser / NeuralFeatureField modules does per image in the reference (main_img_denoising.py:39-47):
 * table U(-1e-4, 1e-4) (tcnn default), nn.Linear default init for the MLPs, G = randn * 0.02 (offline_denoiser.py:33-36). */
int dvt_fit_init_params(dvt_fit_t* h, unsigned long long seed, void* stream);
/* Starts a fit: zeroes Adam state, installs the bank (device, borrowed: feats f32 [rows, C], coords f32 [rows, 2],
 * rows = views*gh*gw, row r belongs to noise-map cell r % (gh*gw)), the sampling stream idx_host int32
 * [num_iters, bsz] (np.random.randint replay; copied before the call returns) and the schedule
 * (adjust_learning_rate, dvt/utils/misc.py:306-322).  freeze_step = int(args.freeze_shared_artifacts_after *
 * args.num_iters), computed by the caller in double like the reference (main_img_denoising.py:70).  validate != 0: the
 * range checks (coordinates in [0, 1] -- the assert of neural_feature_field.py:47 -- and sampled rows inside the bank)
 * are read back and reported by this call (blocks); validate == 0: they are recorded on the device for dvt_fit_check. */
int dvt_fit_begin(dvt_fit_t* h, const float* bank_feats, const float* bank_coords, size_t bank_rows,
                  const int32_t* idx_host, int num_iters, double lr, double min_lr, int warmup_iters, int freeze_step,
                  double weight_decay, double loss_scale, int validate, void* stream);
/* How the shared artifact map G is sampled at the reference's node coordinates (offline_denoiser.py:92-101:
 * F.grid_sample(G, linspace(-1, 1) nodes, bilinear, align_corners=True)).  In fp32 a node's unnormalised position is not
 * always the integer it stands for, so the reference reads -- and sends gradient to -- a neighbouring cell with a weight
 * of ~1e-6; Adam normalises gradients, so this decides the update of cells that were not sampled themselves.  HOST
 * tables of gw + gh entries (x nodes first): first cell, weight of that cell, weight of the next cell, computed by the
 * caller with the reference's own fp32 arithmetic.  Without this call rows are attributed to their cell with weight 1. */
int dvt_fit_set_artifact_grid(dvt_fit_t* h, const int* i0_host, const float* w0_host, const float* w1_host);
/* Reports (and clears) the input-validation result of the fits begun since the last check.  Blocks. */
int dvt_fit_check(dvt_fit_t* h);
/* Runs the next `count` optimisation steps.  graph_steps > 0: CUDA graphs of that many steps. */
int dvt_fit_run(dvt_fit_t* h, int count, int graph_steps, void* stream);
/* Per-step losses, HOST f32 [num_iters, 5]: loss, patch_l2, cosine_similarity, residual, residual_sparsity. */
int dvt_fit_losses(dvt_fit_t* h, float* dst_host, int num_iters);   /* blocks */
/* Same table copied asynchronously on `stream` into pinned-host or device memory. */
int dvt_fit_losses_async(dvt_fit_t* h, float* dst, int num_iters, void* stream);
/* out [n, C] f32 = neural_field(coords [n, 2])  (denoised_feats of the final query, main_img_denoising.py:121-130). */
int dvt_fit_query(dvt_fit_t* h, const float* coords, int n, float* out, void* stream);
/* out [n, C] f32 = residual_predictor(raw [n, C] f32). */
int dvt_fit_residual(dvt_fit_t* h, const float* raw, int n, float* out, void* stream);
/* Measurement hook: ONE dense Adam sweep of the hash table (the dominant HBM-bound kernel of HP-2; reference: the
 * torch.optim.Adam.step() over tcnn's dense table gradient, main_img_denoising.py:88) on `stream`, outside the step
 * schedule.  ctas > 0: that many persistent 1024-thread CTAs (at most one per SM); 0: 8 x #SM CTAs of 256 threads; a
 * negative value is an error.  Modifies the optimiser state -- call after the results of the fit have been read.
 * Requires dvt_fit_begin. */
int dvt_fit_sweep_once(dvt_fit_t* h, int ctas, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Stage 2: training step of the generalizable denoiser (SURVEY.md 8(f-2); reference main_denoiser.py:197-221 -- forward of
 * `Denoiser` (dvt/models/online_denoiser.py:62-104: one pre-LN timm Block), MSE + (1 - cosine) loss, loss.backward(),
 * torch.optim.AdamW.step()).  Unit operators; dvt.models.Denoiser composes them into an autograd function, the forward
 * GEMMs are dvt_gemm_tn / dvt_gemm_tn_residual above.
 * ------------------------------------------------------------------------------------------------------- */
/* Flash-attention backward (replaces autograd through F.scaled_dot_product_attention in timm Attention), head_dim 64 or
 * 80 (D below): dqkv bf16 [B, N, 3*heads*D] from qkv, the forward output `out`, its gradient `dout` (bf16 [B, N,
 * heads*D]) and the lse of dvt_attention_fwd.  Workspaces: dq_workspace f32 [B, N, heads*D], delta_workspace f32
 * [B, heads, N]. */
int dvt_attention_bwd(const void* qkv_bf16, const void* out_bf16, const void* dout_bf16, const float* lse, void* dqkv_bf16,
                      float* dq_workspace, float* delta_workspace, int B, int N, int heads, int head_dim, void* stream);
/* LayerNorm backward: dx_accum [rows, C] += d/dx, dgamma / dbeta [C] += their gradients (all f32; x is the LN input).
 * C % 4 == 0, C <= 2048; x, gamma, dy and dx_accum 16-byte aligned. */
int dvt_layernorm_bwd(const float* x, const float* gamma, const float* dy, float* dx_accum, float* dgamma, float* dbeta,
                      int rows, int C, float eps, void* stream);
/* out_accum[n] += sum_m in[m, n]  (bias gradients); in: bf16 or f32 [rows, cols] with row pitch ld >= cols, 4-byte
 * aligned (bf16: cols and ld even). */
int dvt_colsum(const void* in, int dtype, int ld, int rows, int cols, float* out_accum, void* stream);
/* out = gelu(in), erf form, bf16, n % 8 == 0  (forward of the MLP activation when the pre-activation must be kept). */
int dvt_gelu(const void* in_bf16, void* out_bf16, size_t n, void* stream);
/* Loss of main_denoiser.py:214-217 and its gradient: losses3 = (l2 + cos, l2 = mse, cos = 1 - mean cosine similarity);
 * dpred (optional) = grad_scale * d(l2 + cos)/dpred.  pred, target, dpred f32 [rows, C], 16-byte aligned; C % 4 == 0,
 * C <= 2048. */
int dvt_denoise_loss(const float* pred, const float* target, float* dpred, float* losses3, int rows, int C, float grad_scale,
                     void* stream);
/* torch.optim.AdamW step (main_denoiser.py:176-180,220) over one flat f32 buffer of n (multiple of 4) parameters;
 * step counts from 1.  p, g, m and v 16-byte aligned. */
int dvt_adamw(float* p, const float* g, float* m, float* v, size_t n, double lr, double beta1, double beta2, double eps,
              double weight_decay, long long step, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Stage 3: distillation of the whole ViT backbone (reference main_distillation.py: the student
 * PretrainedViTWrapper is trained so that its features match a frozen Denoiser(vit=...) teacher).  Unit operators that
 * dvt.train_ops composes, with the stage-2 set above, into the autograd graph of the ViT.  The column sums of these
 * calls are fixed-order two-level reductions through `workspace` (f32, at least 256 * C elements), so repeated calls are
 * bit-identical.
 * ------------------------------------------------------------------------------------------------------- */
/* Backward of x += gamma * branch (branch = A.B^T + bias): one pass over dx (f32 [rows, C], row pitch ldx) that writes
 * dbranch = gamma * dx (bf16 [rows, C], optional), dbias[C] = sum_rows gamma * dx and, when dgamma is given, dgamma[C] =
 * sum_rows dx * branch (branch: the bf16 [rows, C] side output of dvt_gemm_tn_residual).  gamma NULL: unit scale (no
 * LayerScale): the call casts dx to bf16 and sums its columns.  dbias / dgamma are overwritten.  C and ldx >= C multiples
 * of 4; dx, gamma and workspace 16-byte aligned, branch and dbranch 8-byte aligned. */
int dvt_layerscale_bwd(const float* dx, int ldx, const void* branch_bf16, const float* gamma, void* dbranch_bf16, float* dbias,
                       float* dgamma, float* workspace, int rows, int C, void* stream);
/* Token assembly of the ViT forward on caller-owned tensors: out [B, prefix + np, C] f32 = patch rows
 * patches (bf16 [B*np, Kp], dvt_im2col) . w^T (bf16 [C, Kp], zero-padded conv weight) + bias + pos_patch[p] after
 * `prefix` rows copied from prefix_rows [prefix, C] (what dvt_vit_forward does before the first block).  bias may be
 * NULL: a patch embedding without bias (the CLIP towers); pos_patch may be NULL: no position term (the RoPE ViTs).
 * out, bias and pos_patch 16-byte aligned. */
int dvt_vit_embed_fwd(const void* patches_bf16, int Kp, const void* w_bf16, const float* bias, const float* pos_patch,
                      const float* prefix_rows, int B, int np, int prefix, int C, float* out, void* stream);
/* Backward of dvt_vit_embed_fwd w.r.t. everything but the image: from dx0 (f32 [B, ntok, C], ntok = prefix + np) writes
 * dpatch (bf16 [B*np, C], the patch rows compacted: the dY of the patch-embed weight gradient), dpos (f32 [np, C], summed
 * over the batch), dprefix (f32 [prefix, C], summed over the batch) and dbias (f32 [C]).  All overwritten.  dx0, dpos,
 * dprefix and workspace 16-byte aligned, dpatch 8-byte aligned. */
int dvt_vit_embed_bwd(const float* dx0, int B, int ntok, int prefix, int C, void* dpatch_bf16, float* dpos, float* dprefix,
                      float* dbias, float* workspace, void* stream);
/* Backward of dvt_layernorm in its in_group / skip form (final norm + prefix strip): dy f32 [rows / in_group * (in_group -
 * skip), C] holds the compacted rows, x and dx_accum f32 [rows, C] the full ones; dx_accum += d/dx on the kept rows only
 * (the skipped rows are not touched); dgamma / dbeta [C] are overwritten.  0 <= skip < in_group, rows % in_group == 0;
 * x, gamma, dy and dx_accum 16-byte aligned. */
int dvt_layernorm_bwd_grouped(const float* x, const float* gamma, const float* dy, float* dx_accum, float* dgamma, float* dbeta,
                              float* workspace, int rows, int C, float eps, int in_group, int skip, void* stream);
/* QKV projection of a RoPE ViT (DINOv3) with the 2-D rotary position embedding in the GEMM epilogue: qkv bf16 [M, 3C]
 * (row pitch ldo >= 3C) = x (bf16 [M, C], pitch ldx) . w^T (bf16 [3C, C], pitch ldw) + bias (f32 [3C], may be NULL); then
 * on the q and k columns (64-wide heads, C = heads * head_dim, head_dim 64) of every row whose token t = m % ntok is a patch
 * token (t >= prefix, patch p = t - prefix), per head and d < 32, in fp32 before the bf16 store:
 *   q[d] <- q[d] cos - q[d + 32] sin,   q[d + 32] <- q[d + 32] cos + q[d] sin,   cos = rope[p, d], sin = rope[p, 32 + d]
 * rope f32 [ntok - prefix, 64] (16-byte aligned; rows (cos | sin) of the angles 2 pi coord_y inv_freq then 2 pi coord_x
 * inv_freq, transformers DINOv3ViTRopePositionEmbedding).  M % ntok == 0, 0 <= prefix < ntok.  The operand and output rules
 * of dvt_gemm_tn apply.  The tensor-core and the SIMT debug kernels (dvt_set_debug_impl) both fuse the rotation.
 * Replaces: q_proj / k_proj / v_proj and apply_rotary_pos_emb of transformers DINOv3ViTAttention. */
int dvt_gemm_qkv_rope(const void* x_bf16, int ldx, const void* w_bf16, int ldw, int M, int C, const float* bias,
                      const float* rope, int ntok, int prefix, int heads, int head_dim, void* qkv_bf16, int ldo, void* stream);
/* Backward of the rotation of dvt_gemm_qkv_rope, in place on the q and k columns of dqkv (bf16 [M, >= 2 * heads * 64], row
 * pitch ld a multiple of 4, 8-byte aligned): on patch rows dx[d] = dy[d] cos + dy[d + 32] sin, dx[d + 32] = dy[d + 32] cos -
 * dy[d] sin (the transpose of the forward rotation; fp32, one bf16 rounding).  Prefix rows and the v columns are not
 * touched.  Same rope table and shape rules as dvt_gemm_qkv_rope; head_dim must be 64.  No reductions: deterministic. */
int dvt_rope_bwd(void* dqkv_bf16, int ld, const float* rope, int M, int ntok, int prefix, int heads, int head_dim,
                 void* stream);
/* SwiGLU MLP (timm SwiGLUPacked, ViT-g/14): out [M, Hh] = silu(g) * u with [g | u] = hpre [M, 2 Hh] (bf16, contiguous), the
 * kernel of the inference forward, so a training forward produces the same bits. */
int dvt_swiglu(const void* hpre_bf16, void* out_bf16, size_t M, int Hh, void* stream);
/* fc2 data gradient of a SwiGLU MLP with the SwiGLU backward fused into the epilogue (the fp32 dh never reaches memory):
 * dh = dy (bf16 [M, K], row pitch ld_dy) . w (fc2 weight, bf16 [K, Hh] in its nn.Linear storage, row pitch ldw), then
 * dhpre[m, n] = dh * u * silu'(g) and dhpre[m, n + Hh] = dh * silu(g), g = hpre[m, n], u = hpre[m, n + Hh] (the saved fc1
 * output).  hpre / dhpre bf16 [M, >= 2 Hh], pitches multiples of 4, 8-byte aligned.  Plain stores: deterministic. */
int dvt_gemm_bf16_dgrad_swiglu(const void* dy_bf16, int ld_dy, const void* w_bf16, int ldw, int M, int Hh, int K,
                               const void* hpre_bf16, int ld_hpre, void* dhpre_bf16, int ld_dhpre, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Deterministic training step (stages 2 and 3 under torch.use_deterministic_algorithms): fixed-order replacements of
 * every float-atomic reduction of the backward.  Same inputs and outputs as the calls they replace; repeated calls on
 * the same GPU model give bit-identical results.  No kernel waits on another CTA.
 * ------------------------------------------------------------------------------------------------------- */
/* dvt_attention_bwd without float atomics: dK / dV come from the same key-major kernel (bit-identical to
 * dvt_attention_bwd's), dQ from a query-major kernel that keeps it in registers over all key tiles and writes it once
 * (bf16).  No dQ workspace; delta_workspace f32 [B, heads, N]. */
int dvt_attention_bwd_det(const void* qkv_bf16, const void* out_bf16, const void* dout_bf16, const float* lse,
                          void* dqkv_bf16, float* delta_workspace, int B, int N, int heads, int head_dim, void* stream);
/* Weight gradient out [M, N] f32 (row pitch ldo, overwritten) = dy^T . x with dy bf16 [K, M] and x bf16 [K, N] read in
 * their [rows, features] storage (row pitches ld_dy, ldx).  splits > 1: split s of the K range writes its partial product
 * with plain stores into plane s of workspace (f32 [splits, M, ldo]), then the planes are added in split order. */
int dvt_gemm_bf16_wgrad_ordered(const void* dy_bf16, int ld_dy, const void* x_bf16, int ldx, int M, int N, int K, float* out,
                                int ldo, int splits, float* workspace, void* stream);
/* out[c] = sum_r in[r, c] (overwritten) in a fixed order; in bf16 or f32 [rows, cols], cols and ld >= cols multiples of 4,
 * in 16-byte (f32) or 8-byte (bf16) aligned; workspace f32 [256 * cols], 16-byte aligned. */
int dvt_colsum_ordered(const void* in, int dtype, int ld, int rows, int cols, float* out, float* workspace, void* stream);
/* dvt_denoise_loss with per-CTA partials added in a fixed order (losses3 overwritten); workspace f32 [2 * ceil(rows / 8)].
 * Same shape and alignment rules as dvt_denoise_loss. */
int dvt_denoise_loss_ordered(const float* pred, const float* target, float* dpred, float* losses3, float* workspace, int rows,
                             int C, float grad_scale, void* stream);
/* Backward of a separable resampling of a [gh, gw, C] grid to [h, w, C] (the bicubic antialiased position-embedding
 * resample) with the forward's fp32 weight matrices wh [h, gh] and ww [w, gw]: dgrid [gh, gw, C] (overwritten) =
 * sum_y sum_x wh[y, i] ww[x, j] dout[y, x, :]; tmp f32 [gh, w, C]. */
int dvt_resample_bwd(const float* wh, const float* ww, const float* dout, float* tmp, float* dgrid, int h, int w, int gh, int gw,
                     int C, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * view generation (SURVEY.md 8(f-1), the step in front of HP-1)
 * Replaces RandomResizedCropFlip.forward (dvt/dataset/transform.py:39-76) + the 8-worker DataLoader of
 * main_img_denoising.py:277-310.  image: device f32 [3, H, W] (already normalised).  boxes_host: HOST int32 [V, 4] =
 * (top, left, height, width) of every crop, flips_host: HOST int32 [V] (the caller draws them with the reference's own
 * RNG calls).  out: device [V, 3, OH, OW] f32 or bf16 = hflip?(resized_crop(image, box, (OH, OW), BICUBIC,
 * antialias=True)); coords_out (optional): device f32 [V, hp, wp, 2] = (x, y) of every patch inside the image.
 * ------------------------------------------------------------------------------------------------------- */
int dvt_view_crops(const float* image, int H, int W, const int* boxes_host, const int* flips_host, int V, void* out,
                   int out_dtype, int OH, int OW, float* coords_out, int hp, int wp, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Dense-task linear probe, semantic segmentation (reference evaluate_dense_tasks.py with the BNHead configs of
 * evaluation/configs/vitb_{voc2012,ade20k}_linear_config.py; mmseg 0.27 EncoderDecoder).  Every resize is ATen's bilinear upsample with
 * align_corners=False, computed in fp32.  No float atomics: repeated calls are bit-identical.
 * ------------------------------------------------------------------------------------------------------- */
/* Training loss of the head and its gradient in one call (replaces mmseg's resize(seg_logit, label size) + CrossEntropyLoss
 * (ignore_index 255, mean over ALL pixels) + their autograd backward).  logits f32 [B, h, w, K] (NHWC), labels u8 [B, H, W];
 * a label >= K (255: ignore) contributes no loss and no gradient.  loss_out f32 [1] = sum over pixels of the cross-entropy
 * of the upsampled logits (overwritten); dlogits f32 [B, h, w, K] (overwritten) = grad_scale * d(loss sum)/d logits at the
 * low resolution.  The full-resolution logits and their gradient are never written.  2 <= K <= 255.
 * workspace f64 [B * ceil(h / 2) * ceil(w / 2)]. */
int dvt_seg_upsample_ce(const float* logits, int B, int h, int w, int K, const uint8_t* labels, int H, int W, float grad_scale,
                        float* loss_out, float* dlogits, double* workspace, void* stream);
/* Slide inference, one window (mmseg EncoderDecoder.slide_inference): upsamples the window's logits f32 [h, w, K] (NHWC) to
 * the window size wh x ww and adds them into acc f32 [K, Hc, Wc] at (y1, x1); count f32 [Hc, Wc] += 1 there.  Windows
 * enqueued in order on one stream add in that order. */
int dvt_seg_slide_accumulate(const float* logits, int h, int w, int K, int y1, int x1, int wh, int ww, float* acc, float* count,
                             int Hc, int Wc, void* stream);
/* Slide inference, end of an image: acc /= count in place, then for every pixel of the original Ho x Wo image the bilinear
 * resize from Hc x Wc, argmax over K (ties: lowest class) and mmseg's intersect_and_union against labels u8 [Ho, Wo]
 * (255 ignored; labels >= K count in the prediction histogram only): hist u64 [4, K] += (intersect, union, pred, label).
 * The resized logits are never written. */
int dvt_seg_predict_hist(float* acc, const float* count, int K, int Hc, int Wc, const uint8_t* labels, int Ho, int Wo,
                         unsigned long long* hist, void* stream);
/* Test-time augmentation (mmseg EncoderDecoder.aug_test), one augmentation: acc f32 [K, Hc, Wc] and count f32 [Hc, Wc]
 * are the augmentation's slide-inference sums (dvt_seg_slide_accumulate; neither is written).  For every pixel of the
 * original Ho x Wo image: the bilinear resize of acc / count from Hc x Wc, softmax over K, un-flipped horizontally when
 * flip != 0, added into prob f32 [K, Ho, Wo].  Each pixel is owned by one CTA: augmentations enqueued in order on one
 * stream add in that order.  K <= 255. */
int dvt_seg_aug_accumulate(const float* acc, const float* count, int K, int Hc, int Wc, int flip, float* prob, int Ho, int Wo,
                           void* stream);
/* Test-time augmentation, end of an image: prob f32 [K, Ho, Wo] (the sum over n_aug augmentations) / n_aug, argmax over
 * K (ties: lowest class) and mmseg's intersect_and_union against labels u8 [Ho, Wo], as dvt_seg_predict_hist:
 * hist u64 [4, K] += (intersect, union, pred, label).  prob is not written. */
int dvt_seg_aug_argmax_hist(const float* prob, int n_aug, int K, const uint8_t* labels, int Ho, int Wo,
                            unsigned long long* hist, void* stream);

/* ---------------------------------------------------------------------------------------------------------
 * Dense-task linear probe, NYU depth (reference evaluation/configs/vitb_nyu_linear_config.py: DepthEncoderDecoder with
 * the BNHead, classify=True, UD bins, linear norm).  Resizes are ATen's bilinear upsample with align_corners=False in fp32.
 * No float atomics: repeated calls are bit-identical.
 * ------------------------------------------------------------------------------------------------------- */
/* Bin-expectation head, forward.  logits f32 [B, h, w, K] (NHWC) are the head's 1x1-conv logits at the feature grid
 * (conv and bilinear upsample commute); bins f32 [K] (device; torch.linspace(min_depth, max_depth, K)).  For every pixel
 * of the (h * up) x (w * up) grid: r = bilinear(logits), a = relu(r) + 0.1, depth = sum_k a_k / sum_j a_j * bins_k.
 * depth f32 [B, h * up, w * up] (overwritten).  1 <= K <= 256. */
int dvt_depth_head_fwd(const float* logits, int B, int h, int w, int K, int up, const float* bins, float* depth, void* stream);
/* Bin-expectation head, backward: ddepth f32 [B, h * up, w * up] -> dlogits f32 [B, h, w, K] (overwritten), gathered
 * per low-resolution cell in a fixed order; d r_k = ddepth (bins_k - depth) / sum_j a_j where r_k > 0, else 0. */
int dvt_depth_head_bwd(const float* logits, int B, int h, int w, int K, int up, const float* bins, const float* ddepth,
                       float* dlogits, void* stream);
/* One-channel bilinear resize in f32 [B, Hi, Wi] -> out [B, Ho, Wo] (overwritten). */
int dvt_depth_resize_fwd(const float* in, int B, int Hi, int Wi, float* out, int Ho, int Wo, void* stream);
/* Its backward in gather form: dout f32 [B, Ho, Wo] -> din f32 [B, Hi, Wi] (overwritten), each input cell summing the
 * output pixels whose taps reach it in row-major order (deterministic, unlike the scatter of F.interpolate). */
int dvt_depth_resize_bwd(const float* dout, int B, int Hi, int Wi, int Ho, int Wo, float* din, void* stream);
/* Whole-image evaluation of one image: maps f32 [n_aug, Hu, Wu] are the head's depth per augmentation (bit a of
 * flip_mask set: augmentation a was flipped horizontally); each is clamped to [min_depth, max_depth], resized to the
 * original Ho x Wo, un-flipped, and the augmentations are averaged in fp32.  Pixels with min_depth < gt < max_depth
 * (gt f32 [Ho, Wo]) inside rows [cy0, cy1) and columns [cx0, cx1) give sums f64 [10] (overwritten) = (count,
 * #ratio < 1.25, < 1.25^2, < 1.25^3, sum |d|/gt, sum d^2/gt, sum d^2, sum err, sum err^2, sum |log10 gt - log10 pred|)
 * with d = gt - pred, err = log pred - log gt.  workspace f64 [1280].  1 <= n_aug <= 32. */
int dvt_depth_eval_sums(const float* maps, int n_aug, unsigned int flip_mask, int Hu, int Wu, const float* gt, int Ho, int Wo,
                        float min_depth, float max_depth, int cy0, int cy1, int cx0, int cx1, double* workspace,
                        double* sums, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DVT_B200_H_ */
