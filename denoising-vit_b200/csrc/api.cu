// extern "C" entry points declared in include/dvt_b200.h.
#include "../../include/dvt_b200.h"

#include "common.cuh"
#include "gemm.cuh"

namespace dvt {
struct Vit;
int vit_create(Vit** out, int embed, int depth, int heads, int patch, int mlp_hidden, int swiglu, int layerscale,
               int prefix, float ln_eps, int pre_norm, int patch_bias, int rope);
void vit_destroy(Vit* v);
int vit_load(Vit* v, const char* name, const float* src, size_t numel);
int vit_reserve(Vit* v, size_t tokens, size_t patches);
int vit_forward(Vit* v, const void* x_in, bool x_bf16, int B, int H, int W, int stride, const float* pos_patch,
                const float* prefix_rows, const float* rope, int layer_index, int apply_norm, float* out, int out_all_tokens,
                cudaStream_t stream);
int vit_forward_layers(Vit* v, const void* x_in, bool x_bf16, int B, int H, int W, int stride, const float* pos_patch,
                       const float* prefix_rows, const float* rope, int n_layers, const int* layers, int apply_norm,
                       float* const* out, int ldo, int out_all_tokens, float* const* prefix_out, cudaStream_t stream);
int vit_patch(const Vit* v);
int vit_prefix(const Vit* v);
struct Fit;
int fit_create(Fit** out, int C, int gh, int gw, int bsz, int n_levels, const float* scale, const uint32_t* res,
               const uint32_t* size, const uint32_t* offset, const uint32_t* hashed);
void fit_destroy(Fit* f);
int fit_set_param(Fit* f, const char* name, const float* src, size_t numel, cudaStream_t caller);
int fit_get_param(Fit* f, const char* name, float* dst, size_t numel);
int fit_init_params(Fit* f, uint64_t seed, cudaStream_t caller);
int fit_begin(Fit* f, const float* bank, const float* coords, size_t bank_rows, const int* idx_host, int num_iters,
              double lr, double min_lr, int warmup_iters, int freeze_step, double weight_decay, double loss_scale,
              int validate, cudaStream_t caller);
int fit_check(Fit* f);
int fit_set_artifact_grid(Fit* f, const int* i0, const float* w0, const float* w1);
int fit_run(Fit* f, int count, int use_graphs, cudaStream_t st);
int fit_losses(Fit* f, float* dst_host, int num_iters);
int fit_losses_async(Fit* f, float* dst, int num_iters, cudaStream_t caller);
int fit_query(Fit* f, const float* coords, int n, float* out, cudaStream_t st);
int fit_residual(Fit* f, const float* raw, int n, float* out, cudaStream_t st);
int fit_sweep_once(Fit* f, int ctas, cudaStream_t st);
int view_crops(const float* image, int H, int W, const int* boxes_host, const int* flips_host, int V, void* out, bool out_bf16,
               int OH, int OW, float* coords_out, int hp, int wp, cudaStream_t st);
int hashgrid_corners(int n_levels, const float* scale, const uint32_t* res, const uint32_t* size, const uint32_t* offset,
                     const uint32_t* hashed, const float* coords, int n, uint32_t* idx, float* w, cudaStream_t st);
int hashgrid_fwd(int n_levels, const float* scale, const uint32_t* res, const uint32_t* size, const uint32_t* offset,
                 const uint32_t* hashed, const float* table, const float* coords, int n, float* out, cudaStream_t st);
int hashgrid_bwd(int n_levels, const float* scale, const uint32_t* res, const uint32_t* size, const uint32_t* offset,
                 const uint32_t* hashed, const float* coords, int n, const float* dout, float* gtable, cudaStream_t st);
int launch_attention_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* out, const __nv_bfloat16* dout, const float* lse,
                         __nv_bfloat16* dqkv, float* dq_acc, float* delta, int B, int N, int heads, cudaStream_t stream,
                         int head_dim);
int launch_rope_bwd(__nv_bfloat16* dqkv, int ld, const float* rope, int M, int ntok, int prefix, int heads, int head_dim,
                    cudaStream_t st);
int launch_layernorm_bwd(const float* x, const float* gamma, const float* dy, float* dx_accum, float* dgamma, float* dbeta,
                         int rows, int C, float eps, cudaStream_t st);
int launch_colsum(const void* in, bool bf16, int ld, int rows, int cols, float* out, cudaStream_t st);
int launch_gelu(const __nv_bfloat16* in, __nv_bfloat16* out, size_t n, cudaStream_t st);
int launch_swiglu(const __nv_bfloat16* hin, __nv_bfloat16* out, size_t M, int Hh, cudaStream_t st);
int launch_denoise_loss(const float* pred, const float* tgt, float* dpred, float* losses, int rows, int C, float grad_scale,
                        cudaStream_t st);
int launch_adamw(float* p, const float* g, float* m, float* v, size_t n, double lr, double beta1, double beta2, double eps,
                 double weight_decay, long long step, cudaStream_t st);
int launch_layerscale_bwd(const float* dx, int ldx, const __nv_bfloat16* branch, const float* gamma, __nv_bfloat16* dbranch,
                          float* dbias, float* dgamma, float* workspace, int rows, int C, cudaStream_t st);
int launch_vit_embed_bwd(const float* dx0, int B, int ntok, int prefix, int C, __nv_bfloat16* dpatch, float* dpos,
                         float* dprefix, float* dbias, float* workspace, cudaStream_t st);
int launch_layernorm_bwd_grouped(const float* x, const float* gamma, const float* dy, float* dx_accum, float* dgamma,
                                 float* dbeta, float* workspace, int rows, int C, float eps, int in_group, int skip,
                                 cudaStream_t st);
int launch_vit_embed_fwd(const __nv_bfloat16* patches, int Kp, const __nv_bfloat16* w, const float* bias, const float* pos_patch,
                         const float* prefix_rows, int B, int np, int prefix, int C, float* out, cudaStream_t st);
int launch_attention_bwd_det(const __nv_bfloat16* qkv, const __nv_bfloat16* out, const __nv_bfloat16* dout, const float* lse,
                             __nv_bfloat16* dqkv, float* delta, int B, int N, int heads, cudaStream_t stream, int head_dim);
int launch_colsum_ordered(const void* in, bool bf16, int ld, int rows, int cols, float* out, float* workspace, cudaStream_t st);
int launch_denoise_loss_ordered(const float* pred, const float* tgt, float* dpred, float* losses, float* workspace, int rows,
                                int C, float grad_scale, cudaStream_t st);
int launch_resample_bwd(const float* wh, const float* ww, const float* dout, float* tmp, float* dgrid, int h, int w, int gh,
                        int gw, int C, cudaStream_t st);
int launch_seg_upsample_ce(const float* logits, int B, int h, int w, int K, const uint8_t* labels, int H, int W,
                           float grad_scale, float* loss_out, float* dlogits, double* workspace, cudaStream_t st);
int launch_seg_slide_accumulate(const float* logits, int h, int w, int K, int y1, int x1, int wh, int ww, float* acc,
                                float* count, int Hc, int Wc, cudaStream_t st);
int launch_seg_predict_hist(float* acc, const float* count, int K, int Hc, int Wc, const uint8_t* labels, int Ho, int Wo,
                            unsigned long long* hist, cudaStream_t st);
int launch_seg_aug_accumulate(const float* acc, const float* count, int K, int Hc, int Wc, int flip, float* prob, int Ho,
                              int Wo, cudaStream_t st);
int launch_seg_aug_argmax_hist(const float* prob, int n_aug, int K, const uint8_t* labels, int Ho, int Wo,
                               unsigned long long* hist, cudaStream_t st);
int launch_depth_head_fwd(const float* logits, int B, int h, int w, int K, int up, const float* bins, float* depth,
                          cudaStream_t st);
int launch_depth_head_bwd(const float* logits, int B, int h, int w, int K, int up, const float* bins, const float* ddepth,
                          float* dlogits, cudaStream_t st);
int launch_depth_resize_fwd(const float* in, int B, int Hi, int Wi, float* out, int Ho, int Wo, cudaStream_t st);
int launch_depth_resize_bwd(const float* dout, int B, int Hi, int Wi, int Ho, int Wo, float* din, cudaStream_t st);
int launch_depth_eval_sums(const float* maps, int n_aug, unsigned int flip_mask, int Hu, int Wu, const float* gt, int Ho,
                           int Wo, float min_depth, float max_depth, int cy0, int cy1, int cx0, int cx1, double* workspace,
                           double* sums, cudaStream_t st);
const char* last_error();
}  // namespace dvt

using namespace dvt;

extern "C" {

int dvt_version(void) { return 104; }

const char* dvt_last_error(void) { return dvt::last_error(); }

int dvt_device_error(unsigned int* code_out) {
  unsigned int v = 0, z = 0;
  cudaError_t e = cudaMemcpyFromSymbol(&v, dvt::g_dvt_dev_error, sizeof(v));
  if (e != cudaSuccess) return dvt::cuda_fail(e, "read device error word", __FILE__, __LINE__);
  if (v) cudaMemcpyToSymbol(dvt::g_dvt_dev_error, &z, sizeof(z));
  if (code_out) *code_out = v;
  return DVT_OK;
}

long long dvt_launch_count(void) { return dvt::launch_count(); }

int dvt_set_debug_impl(int impl) {
  if (impl != 0 && impl != 1 && impl != -1) {
    dvt::set_last_error("dvt_set_debug_impl: impl must be -1, 0 or 1");
    return DVT_ERR_INVALID;
  }
  dvt::set_debug_impl(impl);
  return DVT_OK;
}

int dvt_gemm_tn(const void* A, int lda, const void* B, int ldb, int dtype, int M, int N, int K, const float* bias,
                int act, void* out, int ldo, int out_dtype, int splits, void* stream) {
  DVT_REQUIRE(dtype == DVT_DTYPE_BF16 || dtype == DVT_DTYPE_F32, "dvt_gemm_tn: bad dtype %d", dtype);
  DVT_REQUIRE(out_dtype == DVT_DTYPE_BF16 || out_dtype == DVT_DTYPE_F32, "dvt_gemm_tn: bad out_dtype %d", out_dtype);
  DVT_REQUIRE(A && B && out, "dvt_gemm_tn: null pointer");
  GemmEpi e;
  e.bias = bias;
  e.act = act;
  e.out = out;
  e.ldo = ldo;
  if (splits > 1) {
    // every split runs the epilogue on its partial sum, so a bias would be added once per split
    DVT_REQUIRE(out_dtype == DVT_DTYPE_F32 && act == 0 && bias == nullptr,
                "dvt_gemm_tn: split-K needs fp32 output, no activation and no bias");
    e.out_mode = OUT_F32_ATOMIC;
  } else {
    e.out_mode = out_dtype == DVT_DTYPE_BF16 ? OUT_BF16 : OUT_F32;
  }
  GemmShape s{M, N, K, splits < 1 ? 1 : splits};
  return launch_gemm_tn(A, lda, B, ldb, dtype == DVT_DTYPE_BF16 ? TMAP_BF16 : TMAP_F32, s, e,
                        reinterpret_cast<cudaStream_t>(stream));
}

int dvt_gemm_tn_residual(const void* A, int lda, const void* B, int ldb, int dtype, int M, int N, int K,
                         const float* bias, const float* gamma, float* x_inout, int ldx, void* branch_out_bf16,
                         int ld_branch, void* stream) {
  DVT_REQUIRE(dtype == DVT_DTYPE_BF16 || dtype == DVT_DTYPE_F32, "dvt_gemm_tn_residual: bad dtype %d", dtype);
  DVT_REQUIRE(A && B && x_inout, "dvt_gemm_tn_residual: null pointer");
  DVT_REQUIRE(!branch_out_bf16 || (ld_branch >= N && ld_branch % 4 == 0),
              "dvt_gemm_tn_residual: ld_branch=%d must be >= N=%d and a multiple of 4", ld_branch, N);
  GemmEpi e;
  e.bias = bias;
  e.gamma = gamma;
  e.out = x_inout;
  e.ldo = ldx;
  e.out_mode = OUT_F32_RESID;
  e.branch = reinterpret_cast<__nv_bfloat16*>(branch_out_bf16);
  e.ld_branch = ld_branch;
  GemmShape s{M, N, K, 1};
  return launch_gemm_tn(A, lda, B, ldb, dtype == DVT_DTYPE_BF16 ? TMAP_BF16 : TMAP_F32, s, e,
                        reinterpret_cast<cudaStream_t>(stream));
}

int dvt_layernorm(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int y_dtype,
                  int rows, int C, float eps, int in_group, int skip, void* stream) {
  DVT_REQUIRE(x && gamma && beta && y, "dvt_layernorm: null pointer");
  DVT_REQUIRE(y_dtype == DVT_DTYPE_BF16 || y_dtype == DVT_DTYPE_F32, "dvt_layernorm: bad y_dtype %d", y_dtype);
  return launch_layernorm(x, ldx, gamma, beta, y, ldy, y_dtype == DVT_DTYPE_BF16, rows, C, eps, in_group, skip,
                          reinterpret_cast<cudaStream_t>(stream));
}

int dvt_attention_fwd(const void* qkv_bf16, void* out_bf16, float* lse, int B, int N, int heads, int head_dim,
                      void* stream) {
  DVT_REQUIRE(qkv_bf16 && out_bf16, "dvt_attention_fwd: null pointer");
  return launch_attention(reinterpret_cast<const __nv_bfloat16*>(qkv_bf16), reinterpret_cast<__nv_bfloat16*>(out_bf16),
                          B, N, heads, reinterpret_cast<cudaStream_t>(stream), lse, head_dim);
}

/* ---- stage-2 training operators (SURVEY.md 8(f-2)) ---- */
int dvt_attention_bwd(const void* qkv_bf16, const void* out_bf16, const void* dout_bf16, const float* lse, void* dqkv_bf16,
                      float* dq_workspace, float* delta_workspace, int B, int N, int heads, int head_dim, void* stream) {
  return launch_attention_bwd(reinterpret_cast<const __nv_bfloat16*>(qkv_bf16), reinterpret_cast<const __nv_bfloat16*>(out_bf16),
                              reinterpret_cast<const __nv_bfloat16*>(dout_bf16), lse, reinterpret_cast<__nv_bfloat16*>(dqkv_bf16),
                              dq_workspace, delta_workspace, B, N, heads, reinterpret_cast<cudaStream_t>(stream), head_dim);
}
int dvt_layernorm_bwd(const float* x, const float* gamma, const float* dy, float* dx_accum, float* dgamma, float* dbeta,
                      int rows, int C, float eps, void* stream) {
  return launch_layernorm_bwd(x, gamma, dy, dx_accum, dgamma, dbeta, rows, C, eps, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_colsum(const void* in, int dtype, int ld, int rows, int cols, float* out_accum, void* stream) {
  return launch_colsum(in, dtype == DVT_DTYPE_BF16, ld, rows, cols, out_accum, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_gelu(const void* in_bf16, void* out_bf16, size_t n, void* stream) {
  return launch_gelu(reinterpret_cast<const __nv_bfloat16*>(in_bf16), reinterpret_cast<__nv_bfloat16*>(out_bf16), n,
                     reinterpret_cast<cudaStream_t>(stream));
}
int dvt_gemm_bf16(const void* A, int lda, int a_mn, const void* B, int ldb, int b_mn, int M, int N, int K, void* out,
                  int ldo, int out_dtype, int splits, const void* gelu_preact_bf16, int ld_preact, float* last_col_out,
                  void* stream) {
  DVT_REQUIRE(A && B && out, "dvt_gemm_bf16: null pointer");
  GemmEpi e;
  e.out = out;
  e.ldo = ldo;
  if (splits > 1 || last_col_out) {
    DVT_REQUIRE(out_dtype == DVT_DTYPE_F32 && !gelu_preact_bf16,
                "dvt_gemm_bf16: split-K / last_col_out need plain fp32 output");
    e.out_mode = OUT_F32_ATOMIC;
    e.last_col_out = last_col_out;
  } else {
    e.out_mode = out_dtype == DVT_DTYPE_BF16 ? OUT_BF16 : OUT_F32;
  }
  if (gelu_preact_bf16) {
    e.mask = reinterpret_cast<const __nv_bfloat16*>(gelu_preact_bf16);
    e.ldmask = ld_preact;
    e.mask_mode = 1;
  }
  GemmShape s{M, N, K, splits < 1 ? 1 : splits};
  s.a_mn = a_mn;
  s.b_mn = b_mn;
  return launch_gemm_tn(A, lda, B, ldb, TMAP_BF16, s, e, reinterpret_cast<cudaStream_t>(stream));
}
/* ---- stage-3 (distillation) operators ---- */
int dvt_gemm_qkv_rope(const void* x_bf16, int ldx, const void* w_bf16, int ldw, int M, int C, const float* bias,
                      const float* rope, int ntok, int prefix, int heads, int head_dim, void* qkv_bf16, int ldo, void* stream) {
  DVT_REQUIRE(x_bf16 && w_bf16 && rope && qkv_bf16, "dvt_gemm_qkv_rope: null pointer");
  DVT_REQUIRE(head_dim == 64, "dvt_gemm_qkv_rope: head_dim must be 64 (got %d)", head_dim);
  DVT_REQUIRE(heads > 0 && C == heads * head_dim, "dvt_gemm_qkv_rope: C=%d must be heads * head_dim", C);
  DVT_REQUIRE(ntok > 0 && M % ntok == 0, "dvt_gemm_qkv_rope: M=%d must be a multiple of the tokens per image %d", M, ntok);
  DVT_REQUIRE(ldo >= 3 * C, "dvt_gemm_qkv_rope: ldo=%d must be >= 3C=%d", ldo, 3 * C);
  GemmEpi e;
  e.bias = bias;
  e.out = qkv_bf16;
  e.ldo = ldo;
  e.out_mode = OUT_BF16;
  e.rope = rope;
  e.rope_cols = 2 * C;
  e.rope_ntok = ntok;
  e.rope_prefix = prefix;
  GemmShape s{M, 3 * C, C, 1};
  return launch_gemm_tn(x_bf16, ldx, w_bf16, ldw, TMAP_BF16, s, e, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_rope_bwd(void* dqkv_bf16, int ld, const float* rope, int M, int ntok, int prefix, int heads, int head_dim,
                 void* stream) {
  return launch_rope_bwd(reinterpret_cast<__nv_bfloat16*>(dqkv_bf16), ld, rope, M, ntok, prefix, heads, head_dim,
                         reinterpret_cast<cudaStream_t>(stream));
}
int dvt_swiglu(const void* hpre_bf16, void* out_bf16, size_t M, int Hh, void* stream) {
  return launch_swiglu(reinterpret_cast<const __nv_bfloat16*>(hpre_bf16), reinterpret_cast<__nv_bfloat16*>(out_bf16), M, Hh,
                       reinterpret_cast<cudaStream_t>(stream));
}
int dvt_gemm_bf16_dgrad_swiglu(const void* dy_bf16, int ld_dy, const void* w_bf16, int ldw, int M, int Hh, int K,
                               const void* hpre_bf16, int ld_hpre, void* dhpre_bf16, int ld_dhpre, void* stream) {
  DVT_REQUIRE(dy_bf16 && w_bf16 && hpre_bf16 && dhpre_bf16, "dvt_gemm_bf16_dgrad_swiglu: null pointer");
  GemmEpi e;
  e.out = dhpre_bf16;
  e.ldo = ld_dhpre;
  e.out_mode = OUT_BF16;
  e.mask = reinterpret_cast<const __nv_bfloat16*>(hpre_bf16);
  e.ldmask = ld_hpre;
  e.mask_mode = 2;
  GemmShape s{M, Hh, K, 1};
  s.b_mn = 1;
  return launch_gemm_tn(dy_bf16, ld_dy, w_bf16, ldw, TMAP_BF16, s, e, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_layerscale_bwd(const float* dx, int ldx, const void* branch_bf16, const float* gamma, void* dbranch_bf16, float* dbias,
                       float* dgamma, float* workspace, int rows, int C, void* stream) {
  return launch_layerscale_bwd(dx, ldx, reinterpret_cast<const __nv_bfloat16*>(branch_bf16), gamma,
                               reinterpret_cast<__nv_bfloat16*>(dbranch_bf16), dbias, dgamma, workspace, rows, C,
                               reinterpret_cast<cudaStream_t>(stream));
}
int dvt_vit_embed_fwd(const void* patches_bf16, int Kp, const void* w_bf16, const float* bias, const float* pos_patch,
                      const float* prefix_rows, int B, int np, int prefix, int C, float* out, void* stream) {
  return launch_vit_embed_fwd(reinterpret_cast<const __nv_bfloat16*>(patches_bf16), Kp,
                              reinterpret_cast<const __nv_bfloat16*>(w_bf16), bias, pos_patch, prefix_rows, B, np, prefix, C,
                              out, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_vit_embed_bwd(const float* dx0, int B, int ntok, int prefix, int C, void* dpatch_bf16, float* dpos, float* dprefix,
                      float* dbias, float* workspace, void* stream) {
  return launch_vit_embed_bwd(dx0, B, ntok, prefix, C, reinterpret_cast<__nv_bfloat16*>(dpatch_bf16), dpos, dprefix, dbias,
                              workspace, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_layernorm_bwd_grouped(const float* x, const float* gamma, const float* dy, float* dx_accum, float* dgamma, float* dbeta,
                              float* workspace, int rows, int C, float eps, int in_group, int skip, void* stream) {
  return launch_layernorm_bwd_grouped(x, gamma, dy, dx_accum, dgamma, dbeta, workspace, rows, C, eps, in_group, skip,
                                      reinterpret_cast<cudaStream_t>(stream));
}
int dvt_denoise_loss(const float* pred, const float* target, float* dpred, float* losses3, int rows, int C, float grad_scale,
                     void* stream) {
  return launch_denoise_loss(pred, target, dpred, losses3, rows, C, grad_scale, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_adamw(float* p, const float* g, float* m, float* v, size_t n, double lr, double beta1, double beta2, double eps,
              double weight_decay, long long step, void* stream) {
  return launch_adamw(p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, step, reinterpret_cast<cudaStream_t>(stream));
}

/* ---- deterministic training step (torch.use_deterministic_algorithms) ---- */
int dvt_attention_bwd_det(const void* qkv_bf16, const void* out_bf16, const void* dout_bf16, const float* lse,
                          void* dqkv_bf16, float* delta_workspace, int B, int N, int heads, int head_dim, void* stream) {
  return launch_attention_bwd_det(reinterpret_cast<const __nv_bfloat16*>(qkv_bf16), reinterpret_cast<const __nv_bfloat16*>(out_bf16),
                                  reinterpret_cast<const __nv_bfloat16*>(dout_bf16), lse, reinterpret_cast<__nv_bfloat16*>(dqkv_bf16),
                                  delta_workspace, B, N, heads, reinterpret_cast<cudaStream_t>(stream), head_dim);
}
int dvt_gemm_bf16_wgrad_ordered(const void* dy_bf16, int ld_dy, const void* x_bf16, int ldx, int M, int N, int K, float* out,
                                int ldo, int splits, float* workspace, void* stream) {
  DVT_REQUIRE(dy_bf16 && x_bf16 && out, "dvt_gemm_bf16_wgrad_ordered: null pointer");
  DVT_REQUIRE(splits == 1 || workspace, "dvt_gemm_bf16_wgrad_ordered: split-K needs the workspace");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GemmEpi e;
  e.ldo = ldo;
  GemmShape s{M, N, K, splits < 1 ? 1 : splits};
  s.a_mn = 1;
  s.b_mn = 1;
  if (s.splits == 1) {
    e.out = out;
    e.out_mode = OUT_F32;
    return launch_gemm_tn(dy_bf16, ld_dy, x_bf16, ldx, TMAP_BF16, s, e, st);
  }
  e.out = workspace;
  e.out_mode = OUT_F32_PLANES;
  e.out_plane = (size_t)M * ldo;
  int rc = launch_gemm_tn(dy_bf16, ld_dy, x_bf16, ldx, TMAP_BF16, s, e, st);
  if (rc) return rc;
  return launch_splitk_planes_sum(workspace, s.splits, (size_t)M * ldo, M, N, ldo, out, st);
}
int dvt_colsum_ordered(const void* in, int dtype, int ld, int rows, int cols, float* out, float* workspace, void* stream) {
  return launch_colsum_ordered(in, dtype == DVT_DTYPE_BF16, ld, rows, cols, out, workspace, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_denoise_loss_ordered(const float* pred, const float* target, float* dpred, float* losses3, float* workspace, int rows,
                             int C, float grad_scale, void* stream) {
  return launch_denoise_loss_ordered(pred, target, dpred, losses3, workspace, rows, C, grad_scale,
                                     reinterpret_cast<cudaStream_t>(stream));
}
int dvt_resample_bwd(const float* wh, const float* ww, const float* dout, float* tmp, float* dgrid, int h, int w, int gh, int gw,
                     int C, void* stream) {
  return launch_resample_bwd(wh, ww, dout, tmp, dgrid, h, w, gh, gw, C, reinterpret_cast<cudaStream_t>(stream));
}

int dvt_im2col(const void* x, int x_dtype, void* out_bf16, int B, int H, int W, int P, int S, void* stream) {
  DVT_REQUIRE(x && out_bf16 && P > 0 && S > 0 && H >= P && W >= P, "dvt_im2col: bad arguments");
  const int h = (H - P) / S + 1, w = (W - P) / S + 1, Kp = (3 * P * P + 7) / 8 * 8;
  return launch_im2col(x, x_dtype == DVT_DTYPE_BF16, reinterpret_cast<__nv_bfloat16*>(out_bf16), B, H, W, P, S, h, w, Kp,
                       reinterpret_cast<cudaStream_t>(stream));
}

int dvt_vit_create(dvt_vit_t** out, int embed, int depth, int heads, int patch, int mlp_hidden, int swiglu,
                   int layerscale, int prefix_tokens, float ln_eps, int pre_norm, int patch_bias, int rope) {
  DVT_REQUIRE(out, "dvt_vit_create: null out");
  return vit_create(reinterpret_cast<Vit**>(out), embed, depth, heads, patch, mlp_hidden, swiglu, layerscale,
                    prefix_tokens, ln_eps, pre_norm, patch_bias, rope);
}
void dvt_vit_destroy(dvt_vit_t* h) { vit_destroy(reinterpret_cast<Vit*>(h)); }
int dvt_vit_load(dvt_vit_t* h, const char* timm_key, const float* src, size_t numel) {
  DVT_REQUIRE(h && timm_key && src, "dvt_vit_load: null argument");
  return vit_load(reinterpret_cast<Vit*>(h), timm_key, src, numel);
}
int dvt_vit_reserve(dvt_vit_t* h, int max_batch, int H, int W, int stride) {
  DVT_REQUIRE(h && max_batch > 0 && stride > 0, "dvt_vit_reserve: bad arguments");
  Vit* v = reinterpret_cast<Vit*>(h);
  const int P = vit_patch(v);
  DVT_REQUIRE(H >= P && W >= P, "dvt_vit_reserve: image smaller than a patch");
  const size_t np = (size_t)((H - P) / stride + 1) * ((W - P) / stride + 1);
  return vit_reserve(v, (size_t)max_batch * (np + vit_prefix(v)), (size_t)max_batch * np);
}
int dvt_vit_forward(dvt_vit_t* h, const void* x, int x_dtype, int B, int H, int W, int stride,
                    const float* pos_patch, const float* prefix_rows, const float* rope, int layer_index, int norm, float* out,
                    int all_tokens, void* stream) {
  DVT_REQUIRE(h, "dvt_vit_forward: null handle");
  return vit_forward(reinterpret_cast<Vit*>(h), x, x_dtype == DVT_DTYPE_BF16, B, H, W, stride, pos_patch, prefix_rows, rope,
                     layer_index, norm, out, all_tokens, reinterpret_cast<cudaStream_t>(stream));
}
// Every check that does not need the handle comes before the null-handle check, so that a test without a GPU (no handle can
// be created there) sees each refusal.
int dvt_vit_forward_layers(dvt_vit_t* h, const void* x, int x_dtype, int B, int H, int W, int stride,
                           const float* pos_patch, const float* prefix_rows, const float* rope, int n_layers,
                           const int* layer_indices, int norm, float* const* out, int ldo, int all_tokens,
                           float* const* prefix_out, void* stream) {
  DVT_REQUIRE(x, "dvt_vit_forward_layers: x is null");
  DVT_REQUIRE(prefix_rows, "dvt_vit_forward_layers: prefix_rows is null");
  DVT_REQUIRE(n_layers > 0 && layer_indices, "dvt_vit_forward_layers: layer_indices must list n_layers >= 1 layers (n_layers=%d)",
              n_layers);
  DVT_REQUIRE(layer_indices[0] >= 0, "dvt_vit_forward_layers: layer_indices[0]=%d is negative", layer_indices[0]);
  for (int l = 1; l < n_layers; ++l)
    DVT_REQUIRE(layer_indices[l] > layer_indices[l - 1],
                "dvt_vit_forward_layers: layer_indices must be strictly ascending (layer_indices[%d]=%d after %d)", l,
                layer_indices[l], layer_indices[l - 1]);
  DVT_REQUIRE(ldo > 0 && ldo % 4 == 0, "dvt_vit_forward_layers: ldo=%d must be a positive multiple of 4", ldo);
  DVT_REQUIRE(out, "dvt_vit_forward_layers: out is null");
  for (int l = 0; l < n_layers; ++l) {
    DVT_REQUIRE(out[l], "dvt_vit_forward_layers: out[%d] is null", l);
    DVT_REQUIRE(!misaligned(out[l], 16), "dvt_vit_forward_layers: out[%d] must be 16-byte aligned", l);
  }
  DVT_REQUIRE(!(all_tokens && prefix_out),
              "dvt_vit_forward_layers: prefix_out with all_tokens (out already holds the prefix rows)");
  for (int l = 0; prefix_out && l < n_layers; ++l) {
    DVT_REQUIRE(prefix_out[l], "dvt_vit_forward_layers: prefix_out[%d] is null", l);
    DVT_REQUIRE(!misaligned(prefix_out[l], 16), "dvt_vit_forward_layers: prefix_out[%d] must be 16-byte aligned", l);
  }
  DVT_REQUIRE(h, "dvt_vit_forward_layers: null handle");
  return vit_forward_layers(reinterpret_cast<Vit*>(h), x, x_dtype == DVT_DTYPE_BF16, B, H, W, stride, pos_patch, prefix_rows,
                            rope, n_layers, layer_indices, norm, out, ldo, all_tokens, prefix_out,
                            reinterpret_cast<cudaStream_t>(stream));
}

int dvt_gemm_f32x3(const float* A, int lda, size_t plane_a, int a_mn, const float* B, int ldb, size_t plane_b, int b_mn,
                   int M, int N, int K, float* out, int ldo, int splits, float* last_col_out, void* stream) {
  DVT_REQUIRE(A && B && out, "dvt_gemm_f32x3: null pointer");
  GemmEpi e;
  e.out = out;
  e.ldo = ldo;
  if (splits > 1 || last_col_out) {
    e.out_mode = OUT_F32_ATOMIC;
    e.last_col_out = last_col_out;
  } else {
    e.out_mode = OUT_F32;
  }
  GemmShape s{M, N, K, splits < 1 ? 1 : splits};
  s.a_mn = a_mn; s.b_mn = b_mn; s.x3 = 1; s.plane_a = plane_a; s.plane_b = plane_b;
  return launch_gemm_tn(A, lda, B, ldb, TMAP_F32, s, e, reinterpret_cast<cudaStream_t>(stream));
}

int dvt_hashgrid_corners(int n_levels, const float* scale_host, const uint32_t* res_host, const uint32_t* size_host,
                         const uint32_t* offset_host, const uint32_t* hashed_host, const float* coords, int n,
                         uint32_t* idx_out, float* w_out, void* stream) {
  DVT_REQUIRE(scale_host && res_host && size_host && offset_host && hashed_host && coords && idx_out && w_out && n > 0,
              "dvt_hashgrid_corners: bad arguments");
  return hashgrid_corners(n_levels, scale_host, res_host, size_host, offset_host, hashed_host, coords, n, idx_out, w_out,
                          reinterpret_cast<cudaStream_t>(stream));
}
int dvt_hashgrid_fwd(int n_levels, const float* scale_host, const uint32_t* res_host, const uint32_t* size_host,
                     const uint32_t* offset_host, const uint32_t* hashed_host, const float* table, const float* coords,
                     int n, float* out, void* stream) {
  DVT_REQUIRE(scale_host && res_host && size_host && offset_host && hashed_host && table && coords && out && n > 0,
              "dvt_hashgrid_fwd: bad arguments");
  return hashgrid_fwd(n_levels, scale_host, res_host, size_host, offset_host, hashed_host, table, coords, n, out,
                      reinterpret_cast<cudaStream_t>(stream));
}
int dvt_hashgrid_bwd(int n_levels, const float* scale_host, const uint32_t* res_host, const uint32_t* size_host,
                     const uint32_t* offset_host, const uint32_t* hashed_host, const float* coords, int n,
                     const float* dout, float* grad_table, void* stream) {
  DVT_REQUIRE(scale_host && res_host && size_host && offset_host && hashed_host && coords && dout && grad_table && n > 0,
              "dvt_hashgrid_bwd: bad arguments");
  return hashgrid_bwd(n_levels, scale_host, res_host, size_host, offset_host, hashed_host, coords, n, dout, grad_table,
                      reinterpret_cast<cudaStream_t>(stream));
}

int dvt_fit_create(dvt_fit_t** out, int feat_dim, int gh, int gw, int bsz, int n_levels, const float* scale_host,
                   const uint32_t* res_host, const uint32_t* size_host, const uint32_t* offset_host,
                   const uint32_t* hashed_host) {
  DVT_REQUIRE(out && scale_host && res_host && size_host && offset_host && hashed_host, "dvt_fit_create: null argument");
  return fit_create(reinterpret_cast<Fit**>(out), feat_dim, gh, gw, bsz, n_levels, scale_host, res_host, size_host,
                    offset_host, hashed_host);
}
void dvt_fit_destroy(dvt_fit_t* h) { fit_destroy(reinterpret_cast<Fit*>(h)); }
int dvt_fit_set_param(dvt_fit_t* h, const char* name, const float* src, size_t numel, void* stream) {
  DVT_REQUIRE(h && name && src, "dvt_fit_set_param: null argument");
  return fit_set_param(reinterpret_cast<Fit*>(h), name, src, numel, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_fit_init_params(dvt_fit_t* h, unsigned long long seed, void* stream) {
  DVT_REQUIRE(h, "dvt_fit_init_params: null handle");
  return fit_init_params(reinterpret_cast<Fit*>(h), (uint64_t)seed, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_fit_get_param(dvt_fit_t* h, const char* name, float* dst, size_t numel) {
  DVT_REQUIRE(h && name && dst, "dvt_fit_get_param: null argument");
  return fit_get_param(reinterpret_cast<Fit*>(h), name, dst, numel);
}
int dvt_fit_begin(dvt_fit_t* h, const float* bank_feats, const float* bank_coords, size_t bank_rows,
                  const int32_t* idx_host, int num_iters, double lr, double min_lr, int warmup_iters, int freeze_step,
                  double weight_decay, double loss_scale, int validate, void* stream) {
  DVT_REQUIRE(h, "dvt_fit_begin: null handle");
  return fit_begin(reinterpret_cast<Fit*>(h), bank_feats, bank_coords, bank_rows, idx_host, num_iters, lr, min_lr,
                   warmup_iters, freeze_step, weight_decay, loss_scale, validate, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_fit_set_artifact_grid(dvt_fit_t* h, const int* i0_host, const float* w0_host, const float* w1_host) {
  DVT_REQUIRE(h, "dvt_fit_set_artifact_grid: null handle");
  return fit_set_artifact_grid(reinterpret_cast<Fit*>(h), i0_host, w0_host, w1_host);
}
int dvt_fit_check(dvt_fit_t* h) {
  DVT_REQUIRE(h, "dvt_fit_check: null handle");
  return fit_check(reinterpret_cast<Fit*>(h));
}
int dvt_fit_run(dvt_fit_t* h, int count, int graph_steps, void* stream) {
  DVT_REQUIRE(h, "dvt_fit_run: null handle");
  return fit_run(reinterpret_cast<Fit*>(h), count, graph_steps, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_fit_losses(dvt_fit_t* h, float* dst_host, int num_iters) {
  DVT_REQUIRE(h && dst_host, "dvt_fit_losses: null argument");
  return fit_losses(reinterpret_cast<Fit*>(h), dst_host, num_iters);
}
int dvt_fit_losses_async(dvt_fit_t* h, float* dst, int num_iters, void* stream) {
  DVT_REQUIRE(h && dst, "dvt_fit_losses_async: null argument");
  return fit_losses_async(reinterpret_cast<Fit*>(h), dst, num_iters, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_fit_query(dvt_fit_t* h, const float* coords, int n, float* out, void* stream) {
  DVT_REQUIRE(h, "dvt_fit_query: null handle");
  return fit_query(reinterpret_cast<Fit*>(h), coords, n, out, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_fit_residual(dvt_fit_t* h, const float* raw, int n, float* out, void* stream) {
  DVT_REQUIRE(h, "dvt_fit_residual: null handle");
  return fit_residual(reinterpret_cast<Fit*>(h), raw, n, out, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_fit_sweep_once(dvt_fit_t* h, int ctas, void* stream) {
  DVT_REQUIRE(h, "dvt_fit_sweep_once: null handle");
  return fit_sweep_once(reinterpret_cast<Fit*>(h), ctas, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_view_crops(const float* image, int H, int W, const int* boxes_host, const int* flips_host, int V, void* out,
                   int out_dtype, int OH, int OW, float* coords_out, int hp, int wp, void* stream) {
  return view_crops(image, H, W, boxes_host, flips_host, V, out, out_dtype == DVT_DTYPE_BF16, OH, OW, coords_out, hp, wp,
                    reinterpret_cast<cudaStream_t>(stream));
}

int dvt_seg_upsample_ce(const float* logits, int B, int h, int w, int K, const uint8_t* labels, int H, int W, float grad_scale,
                        float* loss_out, float* dlogits, double* workspace, void* stream) {
  return launch_seg_upsample_ce(logits, B, h, w, K, labels, H, W, grad_scale, loss_out, dlogits, workspace,
                                reinterpret_cast<cudaStream_t>(stream));
}
int dvt_seg_slide_accumulate(const float* logits, int h, int w, int K, int y1, int x1, int wh, int ww, float* acc, float* count,
                             int Hc, int Wc, void* stream) {
  return launch_seg_slide_accumulate(logits, h, w, K, y1, x1, wh, ww, acc, count, Hc, Wc,
                                     reinterpret_cast<cudaStream_t>(stream));
}
int dvt_seg_predict_hist(float* acc, const float* count, int K, int Hc, int Wc, const uint8_t* labels, int Ho, int Wo,
                         unsigned long long* hist, void* stream) {
  return launch_seg_predict_hist(acc, count, K, Hc, Wc, labels, Ho, Wo, hist, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_seg_aug_accumulate(const float* acc, const float* count, int K, int Hc, int Wc, int flip, float* prob, int Ho, int Wo,
                           void* stream) {
  return launch_seg_aug_accumulate(acc, count, K, Hc, Wc, flip, prob, Ho, Wo, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_seg_aug_argmax_hist(const float* prob, int n_aug, int K, const uint8_t* labels, int Ho, int Wo,
                            unsigned long long* hist, void* stream) {
  return launch_seg_aug_argmax_hist(prob, n_aug, K, labels, Ho, Wo, hist, reinterpret_cast<cudaStream_t>(stream));
}

int dvt_depth_head_fwd(const float* logits, int B, int h, int w, int K, int up, const float* bins, float* depth, void* stream) {
  return launch_depth_head_fwd(logits, B, h, w, K, up, bins, depth, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_depth_head_bwd(const float* logits, int B, int h, int w, int K, int up, const float* bins, const float* ddepth,
                       float* dlogits, void* stream) {
  return launch_depth_head_bwd(logits, B, h, w, K, up, bins, ddepth, dlogits, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_depth_resize_fwd(const float* in, int B, int Hi, int Wi, float* out, int Ho, int Wo, void* stream) {
  return launch_depth_resize_fwd(in, B, Hi, Wi, out, Ho, Wo, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_depth_resize_bwd(const float* dout, int B, int Hi, int Wi, int Ho, int Wo, float* din, void* stream) {
  return launch_depth_resize_bwd(dout, B, Hi, Wi, Ho, Wo, din, reinterpret_cast<cudaStream_t>(stream));
}
int dvt_depth_eval_sums(const float* maps, int n_aug, unsigned int flip_mask, int Hu, int Wu, const float* gt, int Ho, int Wo,
                        float min_depth, float max_depth, int cy0, int cy1, int cx0, int cx1, double* workspace,
                        double* sums, void* stream) {
  return launch_depth_eval_sums(maps, n_aug, flip_mask, Hu, Wu, gt, Ho, Wo, min_depth, max_depth, cy0, cy1, cx0, cx1,
                                workspace, sums, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
