// HP-1: frozen-ViT forward that produces per-patch feature maps.
// Replaces `PretrainedViTWrapper.get_intermediate_layers` -> timm `forward_intermediates`
// (dvt/models/vit_wrapper.py:122-143) for the standard pre-LN ViT family (DINOv2 S/B/L/g, +reg4).
//
// Data flow per call (M = B * tokens, C = embed dim), all activations resident in HBM workspaces owned by the
// handle; the residual stream is fp32, GEMM operands bf16 with fp32 accumulation in registers (wgmma):
//   im2col -> [GEMM patch-embed (+ bias) + pos-embed -> x] -> prefix rows [-> norm_pre LayerNorm (CLIP: pre_norm)]
//   per block: LN1 -> [GEMM qkv + bias] -> attention -> [GEMM proj + bias, x += ls1 * .] ->
//              LN2 -> [GEMM fc1 + bias + GELU] -> [GEMM fc2 + bias, x += ls2 * .]
//   final LayerNorm + prefix strip -> NHWC fp32 (the layout main_img_denoising.py:323 permutes to)
// Blocks after `layer_index` are skipped: the reference runs them (no stop_early) but they cannot change the
// requested output.
#include "common.cuh"

#include <cstdlib>
#include "gemm.cuh"

#include <string>
#include <vector>

namespace dvt {

int launch_layernorm(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, bool out_bf16,
                     int rows, int C, float eps, int in_group, int skip, cudaStream_t stream);
int launch_im2col(const void* x, bool x_bf16, __nv_bfloat16* out, int B, int H, int W, int P, int S, int h, int w,
                  int Kp, cudaStream_t stream);
int launch_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int N, int heads, cudaStream_t stream,
                     int impl, float* lse = nullptr, int head_dim = 64);
__global__ void strip_copy_kernel(const float*, int, float*, int, int, int, int, int);
__global__ void prefix_rows_kernel(const float*, float*, int, int, int, int);
__global__ void swiglu_kernel(const __nv_bfloat16*, __nv_bfloat16*, size_t, int);
__global__ void cast_f32_bf16_kernel(const float*, __nv_bfloat16*, size_t);
__global__ void pad_cast_rows_kernel(const float*, int, __nv_bfloat16*, int, size_t);

struct VitBlock {
  float *n1w = nullptr, *n1b = nullptr, *qkv_b = nullptr, *proj_b = nullptr, *ls1 = nullptr;
  float *n2w = nullptr, *n2b = nullptr, *fc1_b = nullptr, *fc2_b = nullptr, *ls2 = nullptr;
  __nv_bfloat16 *qkv_w = nullptr, *proj_w = nullptr, *fc1_w = nullptr, *fc2_w = nullptr;
};

struct Vit {
  int embed, depth, heads, patch, mlp_hidden, swiglu, layerscale, prefix;
  int head_dim, pre_norm, patch_bias;
  float ln_eps;
  int Kp;  // padded patch-embed K
  __nv_bfloat16* pe_w = nullptr;
  float *pe_b = nullptr, *norm_w = nullptr, *norm_b = nullptr;
  float *npre_w = nullptr, *npre_b = nullptr;  // norm_pre (pre_norm only)
  std::vector<VitBlock> blocks;
  std::vector<void*> owned;
  // workspace
  size_t cap_tokens = 0, cap_patches = 0;
  float* x = nullptr;
  float* x_embed = nullptr;  // token assembly output when pre_norm (norm_pre then writes x)
  __nv_bfloat16 *xn = nullptr, *qkv = nullptr, *attn = nullptr, *hid = nullptr, *hid2 = nullptr, *patches = nullptr;
  float* stage = nullptr;
  size_t stage_cap = 0;
  int loaded = 0;
};

static int dev_alloc(Vit* v, void** p, size_t bytes) {
  DVT_CUDA_OK(cudaMalloc(p, bytes));
  v->owned.push_back(*p);
  return DVT_OK;
}

int vit_create(Vit** out, int embed, int depth, int heads, int patch, int mlp_hidden, int swiglu, int layerscale,
               int prefix, float ln_eps, int pre_norm, int patch_bias) {
  {
    int prc = gemm_prepare();
    if (prc) return prc;
  }
  DVT_REQUIRE(heads > 0 && (embed == heads * 64 || embed == heads * 80),
              "vit: head_dim must be 64 or 80 (embed=%d heads=%d)", embed, heads);
  DVT_REQUIRE(embed % 8 == 0 && mlp_hidden % 8 == 0 && depth > 0 && patch > 0 && prefix >= 1, "vit: bad config");
  Vit* v = new Vit();
  v->embed = embed; v->depth = depth; v->heads = heads; v->patch = patch; v->mlp_hidden = mlp_hidden;
  v->swiglu = swiglu; v->layerscale = layerscale; v->prefix = prefix; v->ln_eps = ln_eps;
  v->head_dim = embed / heads; v->pre_norm = pre_norm ? 1 : 0; v->patch_bias = patch_bias ? 1 : 0;
  v->Kp = (3 * patch * patch + 7) / 8 * 8;
  v->blocks.resize(depth);
  const int C = embed, Hm = mlp_hidden, fc2_in = swiglu ? mlp_hidden / 2 : mlp_hidden;
  int rc = 0;
  auto A = [&](void** p, size_t bytes) { if (!rc) rc = dev_alloc(v, p, bytes); };
  A((void**)&v->pe_w, (size_t)C * v->Kp * 2);
  A((void**)&v->pe_b, C * 4); A((void**)&v->norm_w, C * 4); A((void**)&v->norm_b, C * 4);
  if (v->pre_norm) { A((void**)&v->npre_w, C * 4); A((void**)&v->npre_b, C * 4); }
  for (auto& b : v->blocks) {
    A((void**)&b.n1w, C * 4); A((void**)&b.n1b, C * 4); A((void**)&b.n2w, C * 4); A((void**)&b.n2b, C * 4);
    A((void**)&b.qkv_b, 3 * C * 4); A((void**)&b.proj_b, C * 4); A((void**)&b.fc1_b, Hm * 4); A((void**)&b.fc2_b, C * 4);
    A((void**)&b.ls1, C * 4); A((void**)&b.ls2, C * 4);
    A((void**)&b.qkv_w, (size_t)3 * C * C * 2); A((void**)&b.proj_w, (size_t)C * C * 2);
    A((void**)&b.fc1_w, (size_t)Hm * C * 2); A((void**)&b.fc2_w, (size_t)C * fc2_in * 2);
  }
  if (rc) { for (void* p : v->owned) cudaFree(p); delete v; return rc; }
  *out = v;
  return DVT_OK;
}

void vit_destroy(Vit* v) {
  if (!v) return;
  for (void* p : v->owned) cudaFree(p);
  cudaFree(v->x); cudaFree(v->xn); cudaFree(v->qkv); cudaFree(v->attn); cudaFree(v->hid); cudaFree(v->hid2);
  cudaFree(v->x_embed); cudaFree(v->patches); cudaFree(v->stage);
  delete v;
}

// name: timm state-dict key without the wrapper's "model." prefix.  src: fp32, host or device memory.
int vit_load(Vit* v, const char* name_c, const float* src, size_t numel) {
  const std::string name(name_c);
  const int C = v->embed, Hm = v->mlp_hidden, fc2_in = v->swiglu ? Hm / 2 : Hm;
  float* f32_dst = nullptr;
  __nv_bfloat16* bf_dst = nullptr;
  size_t expect = 0;
  bool pad_pe = false;
  if (name == "patch_embed.proj.weight") { bf_dst = v->pe_w; expect = (size_t)C * 3 * v->patch * v->patch; pad_pe = true; }
  else if (name == "patch_embed.proj.bias" && v->patch_bias) { f32_dst = v->pe_b; expect = C; }
  else if (name == "norm_pre.weight" && v->pre_norm) { f32_dst = v->npre_w; expect = C; }
  else if (name == "norm_pre.bias" && v->pre_norm) { f32_dst = v->npre_b; expect = C; }
  else if (name == "norm.weight") { f32_dst = v->norm_w; expect = C; }
  else if (name == "norm.bias") { f32_dst = v->norm_b; expect = C; }
  else if (name.rfind("blocks.", 0) == 0) {
    size_t dot = name.find('.', 7);
    DVT_REQUIRE(dot != std::string::npos, "vit_load: bad key %s", name_c);
    int i = atoi(name.substr(7, dot - 7).c_str());
    DVT_REQUIRE(i >= 0 && i < v->depth, "vit_load: block index out of range in %s", name_c);
    VitBlock& b = v->blocks[i];
    const std::string k = name.substr(dot + 1);
    if (k == "norm1.weight") { f32_dst = b.n1w; expect = C; }
    else if (k == "norm1.bias") { f32_dst = b.n1b; expect = C; }
    else if (k == "norm2.weight") { f32_dst = b.n2w; expect = C; }
    else if (k == "norm2.bias") { f32_dst = b.n2b; expect = C; }
    else if (k == "attn.qkv.weight") { bf_dst = b.qkv_w; expect = (size_t)3 * C * C; }
    else if (k == "attn.qkv.bias") { f32_dst = b.qkv_b; expect = 3 * C; }
    else if (k == "attn.proj.weight") { bf_dst = b.proj_w; expect = (size_t)C * C; }
    else if (k == "attn.proj.bias") { f32_dst = b.proj_b; expect = C; }
    else if (k == "ls1.gamma") { f32_dst = b.ls1; expect = C; }
    else if (k == "ls2.gamma") { f32_dst = b.ls2; expect = C; }
    else if (k == "mlp.fc1.weight") { bf_dst = b.fc1_w; expect = (size_t)Hm * C; }
    else if (k == "mlp.fc1.bias") { f32_dst = b.fc1_b; expect = Hm; }
    else if (k == "mlp.fc2.weight") { bf_dst = b.fc2_w; expect = (size_t)C * fc2_in; }
    else if (k == "mlp.fc2.bias") { f32_dst = b.fc2_b; expect = C; }
  }
  DVT_REQUIRE(f32_dst || bf_dst, "vit_load: unknown key %s", name_c);
  DVT_REQUIRE(numel == expect, "vit_load: %s has %zu elements, expected %zu", name_c, numel, expect);
  if (f32_dst) {
    DVT_CUDA_OK(cudaMemcpy(f32_dst, src, numel * 4, cudaMemcpyDefault));
  } else {
    if (v->stage_cap < numel) {
      cudaFree(v->stage);
      v->stage = nullptr; v->stage_cap = 0;
      DVT_CUDA_OK(cudaMalloc(&v->stage, numel * 4));
      v->stage_cap = numel;
    }
    DVT_CUDA_OK(cudaMemcpy(v->stage, src, numel * 4, cudaMemcpyDefault));
    if (pad_pe) {
      const size_t total = (size_t)C * v->Kp;
      pad_cast_rows_kernel<<<(unsigned)((total + 255) / 256), 256>>>(v->stage, 3 * v->patch * v->patch, bf_dst, v->Kp, C);
    } else {
      cast_f32_bf16_kernel<<<(unsigned)((numel + 255) / 256 < 65535 ? (numel + 255) / 256 : 65535), 256>>>(v->stage, bf_dst, numel);
    }
    DVT_CUDA_OK(cudaGetLastError());
    DVT_CUDA_OK(cudaDeviceSynchronize());
  }
  v->loaded++;
  return DVT_OK;
}

int vit_patch(const Vit* v) { return v->patch; }
int vit_prefix(const Vit* v) { return v->prefix; }

int vit_reserve(Vit* v, size_t tokens, size_t patches) {
  const int C = v->embed;
  if (tokens > v->cap_tokens) {
    cudaFree(v->x); cudaFree(v->xn); cudaFree(v->qkv); cudaFree(v->attn); cudaFree(v->hid); cudaFree(v->hid2);
    cudaFree(v->x_embed);
    v->x = v->x_embed = nullptr; v->xn = v->qkv = v->attn = v->hid = v->hid2 = nullptr; v->cap_tokens = 0;
    DVT_CUDA_OK(cudaMalloc(&v->x, tokens * C * 4));
    if (v->pre_norm) DVT_CUDA_OK(cudaMalloc(&v->x_embed, tokens * C * 4));
    DVT_CUDA_OK(cudaMalloc(&v->xn, tokens * C * 2));
    DVT_CUDA_OK(cudaMalloc(&v->qkv, tokens * 3 * C * 2));
    DVT_CUDA_OK(cudaMalloc(&v->attn, tokens * C * 2));
    DVT_CUDA_OK(cudaMalloc(&v->hid, tokens * (size_t)v->mlp_hidden * 2));
    if (v->swiglu) DVT_CUDA_OK(cudaMalloc(&v->hid2, tokens * (size_t)(v->mlp_hidden / 2) * 2));
    v->cap_tokens = tokens;
  }
  if (patches > v->cap_patches) {
    cudaFree(v->patches); v->patches = nullptr; v->cap_patches = 0;
    DVT_CUDA_OK(cudaMalloc(&v->patches, patches * v->Kp * 2));
    v->cap_patches = patches;
  }
  return DVT_OK;
}

int vit_forward(Vit* v, const void* x_in, bool x_bf16, int B, int H, int W, int stride, const float* pos_patch,
                const float* prefix_rows, int layer_index, int apply_norm, float* out, int out_all_tokens,
                cudaStream_t stream, int impl) {
  const int C = v->embed, P = v->patch;
  DVT_REQUIRE(B > 0 && H >= P && W >= P && stride > 0, "vit_forward: bad input shape B=%d H=%d W=%d stride=%d", B, H, W, stride);
  DVT_REQUIRE(layer_index >= 0 && layer_index < v->depth, "vit_forward: layer_index %d out of range", layer_index);
  DVT_REQUIRE(pos_patch && prefix_rows && out && x_in, "vit_forward: null pointer");
  const int h = (H - P) / stride + 1, w = (W - P) / stride + 1;
  const int np = h * w, ntok = np + v->prefix;
  const size_t M = (size_t)B * ntok;
  DVT_REQUIRE(M < (size_t)1 << 30, "vit_forward: too many tokens");
  int rc = vit_reserve(v, M, (size_t)B * np);
  if (rc) return rc;
  const int gi = impl;  // gemm / attention implementation selector (-1 default)

  rc = launch_im2col(x_in, x_bf16, v->patches, B, H, W, P, stride, h, w, v->Kp, stream);
  if (rc) return rc;
  float* x_tok = v->pre_norm ? v->x_embed : v->x;  // token assembly target
  {
    GemmEpi e;
    e.bias = v->patch_bias ? v->pe_b : nullptr; e.out_mode = OUT_F32_REMAP; e.out = x_tok; e.ldo = C; e.addend = pos_patch;
    e.rows_per_group = np; e.group_stride = ntok; e.row_offset = v->prefix;
    GemmShape s{B * np, C, v->Kp, 1};
    rc = launch_gemm_tn(v->patches, v->Kp, v->pe_w, v->Kp, TMAP_BF16, s, e, stream, gi);
    if (rc) return rc;
  }
  prefix_rows_kernel<<<B * v->prefix, 256, 0, stream>>>(prefix_rows, x_tok, B, v->prefix, ntok, C);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  if (v->pre_norm) {  // timm norm_pre over every token row (f32 -> f32, out of place)
    rc = launch_layernorm(v->x_embed, C, v->npre_w, v->npre_b, v->x, C, false, (int)M, C, v->ln_eps, 1, 0, stream);
    if (rc) return rc;
  }

  const int Mi = (int)M;
  // Programmatic dependent launch along the block stack is available (DVT_VIT_PDL=1) but OFF by default: these kernels
  // are long, so the hidden launch latency is worth little, and CTAs that are resident early but blocked in
  // griddepcontrol.wait take SM slots from the fit running beside the forwards.  The fit's short kernels are where PDL
  // pays (fit.cu).
  static int vit_pdl = -1;
  if (vit_pdl < 0) {
    const char* pv = getenv("DVT_VIT_PDL");
    vit_pdl = (pv && pv[0] == '1') ? 1 : 0;
  }
  struct PdlScope {
    PdlScope(bool on) { g_vit_pdl = on; }
    ~PdlScope() { g_vit_pdl = false; }
  } pdl_scope(vit_pdl != 0);
  for (int i = 0; i <= layer_index; ++i) {
    const VitBlock& b = v->blocks[i];
    rc = launch_layernorm(v->x, C, b.n1w, b.n1b, v->xn, C, true, Mi, C, v->ln_eps, 1, 0, stream);
    if (rc) return rc;
    {
      GemmEpi e; e.bias = b.qkv_b; e.out_mode = OUT_BF16; e.out = v->qkv; e.ldo = 3 * C;
      GemmShape s{Mi, 3 * C, C, 1};
      s.pdl = vit_pdl;
      rc = launch_gemm_tn(v->xn, C, b.qkv_w, C, TMAP_BF16, s, e, stream, gi);
      if (rc) return rc;
    }
    rc = launch_attention(v->qkv, v->attn, B, ntok, v->heads, stream, gi < 0 ? default_gemm_impl() : gi, nullptr,
                          v->head_dim);
    if (rc) return rc;
    {
      GemmEpi e; e.bias = b.proj_b; e.out_mode = OUT_F32_RESID; e.out = v->x; e.ldo = C;
      e.gamma = v->layerscale ? b.ls1 : nullptr;
      GemmShape s{Mi, C, C, 1};
      s.pdl = vit_pdl;
      rc = launch_gemm_tn(v->attn, C, b.proj_w, C, TMAP_BF16, s, e, stream, gi);
      if (rc) return rc;
    }
    rc = launch_layernorm(v->x, C, b.n2w, b.n2b, v->xn, C, true, Mi, C, v->ln_eps, 1, 0, stream);
    if (rc) return rc;
    const __nv_bfloat16* fc2_in = v->hid;
    int fc2_k = v->mlp_hidden;
    {
      GemmEpi e; e.bias = b.fc1_b; e.act = v->swiglu ? ACT_NONE : ACT_GELU; e.out_mode = OUT_BF16; e.out = v->hid;
      e.ldo = v->mlp_hidden;
      GemmShape s{Mi, v->mlp_hidden, C, 1};
      s.pdl = vit_pdl;
      rc = launch_gemm_tn(v->xn, C, b.fc1_w, C, TMAP_BF16, s, e, stream, gi);
      if (rc) return rc;
    }
    if (v->swiglu) {
      fc2_k = v->mlp_hidden / 2;
      swiglu_kernel<<<num_sms() * 8, 256, 0, stream>>>(v->hid, v->hid2, M, fc2_k);
      DVT_CUDA_OK(cudaGetLastError());
      count_launch();
      fc2_in = v->hid2;
    }
    {
      GemmEpi e; e.bias = b.fc2_b; e.out_mode = OUT_F32_RESID; e.out = v->x; e.ldo = C;
      e.gamma = v->layerscale ? b.ls2 : nullptr;
      GemmShape s{Mi, C, fc2_k, 1};
      s.pdl = vit_pdl;
      rc = launch_gemm_tn(fc2_in, fc2_k, b.fc2_w, fc2_k, TMAP_BF16, s, e, stream, gi);
      if (rc) return rc;
    }
  }
  const int skip = out_all_tokens ? 0 : v->prefix;
  if (apply_norm) {
    rc = launch_layernorm(v->x, C, v->norm_w, v->norm_b, out, C, false, Mi, C, v->ln_eps, ntok, skip, stream);
    if (rc) return rc;
  } else {
    strip_copy_kernel<<<Mi, 256, 0, stream>>>(v->x, C, out, C, Mi, C, ntok, skip);
    DVT_CUDA_OK(cudaGetLastError());
    count_launch();
  }
  return DVT_OK;
}

}  // namespace dvt
