// Shared declarations for the TN GEMM (C[M,N] = A[M,K] * B[N,K]^T, both operands K-contiguous) and its
// fused epilogues.  Used by the ViT forward (HP-1) and by the neural-field fit (HP-2).
#pragma once
#include "common.cuh"

namespace dvt {

enum GemmAct { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2 };
enum GemmOut {
  OUT_BF16 = 0,        // out[m, n] = v                     (bf16)
  OUT_F32 = 1,         // out[m, n] = v                     (fp32)
  OUT_F32_ATOMIC = 2,  // out[m, n] += v                    (fp32 atomics; split-K partial sums)
  OUT_F32_RESID = 3,   // out[m, n] += gamma[n] * v         (fp32 residual stream, in place; gamma may be null)
  OUT_F32_REMAP = 4,   // out[remap(m), n] = v + addend[m % rows_per_group, n]   (patch-embed -> token rows)
  OUT_F32_SPLIT = 5,   // out[m, n] = tf32_hi(v), out[out_plane + m*ldo + n] = v - tf32_hi(v)   (operand of an x3 GEMM)
  OUT_F32_PLANES = 6,  // out[split * out_plane + m*ldo + n] = v   (split-K partials, plain stores, one plane per split;
                       // bf16 wgmma with both operands MN-major only: its own kernel, gemm.cu)
};

// fp32 value -> (hi, lo) with hi exactly representable in TF32 (low 13 mantissa bits zero) and hi + lo == v exactly
__device__ __forceinline__ float tf32_hi(float v) { return __uint_as_float(__float_as_uint(v) & 0xFFFFE000u); }

struct GemmEpi {
  // pre-stage (per element, thread-per-row registers)
  const float* bias = nullptr;        // [N] added to the accumulator
  int act = ACT_NONE;                 // activation applied after bias
  const __nv_bfloat16* mask = nullptr;  // optional [M, ldmask]: v *= (mask[m, n] > 0)   (ReLU backward)
  const float* mask_f32 = nullptr;      // same, fp32 mask tensor
  int ldmask = 0;
  int mask_mode = 0;                  // bf16 `mask` only: 0 = gate (v *= mask > 0), 1 = v *= gelu'(mask)  (GELU backward:
                                      // `mask` holds the pre-activation of the forward pass), 2 = SwiGLU backward (`mask`
                                      // = [g | u] of width 2N, bf16 output of width 2N; its own kernel, gemm.cu)
  float alpha = 1.0f;                 // v *= alpha (after activation / mask)
  // post-stage (coalesced)
  int out_mode = OUT_BF16;
  void* out = nullptr;
  int ldo = 0;
  size_t out_plane = 0;               // OUT_F32_SPLIT: element offset of the lo plane; OUT_F32_PLANES: between split planes
  unsigned long long* entry_guard = nullptr;  // always null: register allocation aid, see gemm_entry_guard (gemm.cu)
  int last_col_n = -1;                // = N-1 when last_col_out is set (filled in by launch_gemm)
  float* last_col_out = nullptr;      // OUT_F32_ATOMIC only: column N-1 is accumulated into last_col_out[m] instead
                                      // (bias gradient through a ones column in the B operand)
  const float* gamma = nullptr;       // LayerScale (OUT_F32_RESID)
  __nv_bfloat16* branch = nullptr;    // OUT_F32_RESID only, optional [M, ld_branch]: the pre-LayerScale value v (bf16), kept
  int ld_branch = 0;                  // for the LayerScale gradient (training forward of the ViT)
  const float* addend = nullptr;      // [rows_per_group, N] (OUT_F32_REMAP)
  int rows_per_group = 0;             // patches per image
  int group_stride = 0;               // tokens per image
  int row_offset = 0;                 // prefix tokens
  unsigned* splitk_sem = nullptr;     // OUT_F32_ATOMIC with split-K, 3xTF32 kernel: one zeroed counter per output tile; the
                                      // splits of a tile then add in split order (a deterministic sum), resetting it to 0
  float* out_t = nullptr;             // OUT_F32_SPLIT of a 3xTF32 product with both operands K-major (and the SIMT debug
  int ldt = 0;                        // GEMM), optional: the same hi / lo values transposed, out_t[n * ldt + m] = hi,
  size_t plane_t = 0;                 // out_t[plane_t + n * ldt + m] = lo (the K-major operand of a later product over m)
  // 2-D rotary position embedding of a QKV projection (OUT_BF16, bf16 operands both K-major, no split-K): columns
  // [0, rope_cols) are 64-wide heads (q then k); in row m, token t = m % rope_ntok, the patch rows t >= rope_prefix get
  //   out[d] = v[d] cos - v[d + 32] sin,  out[d + 32] = v[d + 32] cos + v[d] sin   (d < 32, v = acc + bias, fp32)
  // with cos = rope[p * 64 + d], sin = rope[p * 64 + 32 + d], p = t - rope_prefix.  Its own kernel (gemm.cu).
  const float* rope = nullptr;
  int rope_cols = 0;
  int rope_ntok = 0;
  int rope_prefix = 0;
};

struct GemmShape {
  int M, N, K;
  int splits;    // split-K factor (>1 requires OUT_F32_ATOMIC)
  int a_mn = 0;  // 0: A is [M, K] row-major (K contiguous);  1: A is stored as [K, M] row-major (M contiguous)
  int b_mn = 0;  // 0: B is [N, K] row-major (K contiguous);  1: B is stored as [K, N] row-major (N contiguous)
  // 3xTF32 ("x3"): fp32-accurate product on the tensor cores.  Each fp32 operand is stored as two planes
  // (hi = TF32-exact part at the base pointer, lo = remainder at base + plane elements) and the kernel accumulates
  // A_hi.B_hi + A_hi.B_lo + A_lo.B_hi.
  int x3 = 0;    // 1: 3xTF32 as described
  size_t plane_a = 0, plane_b = 0;
  int pdl = 0;   // launch with programmatic stream serialisation (the kernel calls pdl_wait() after its set-up)
};

// FIT = true (the 3xTF32 kernels of the stage-1 fit): epilogue features only other callers use -- GELU, the bf16 mask with
// GELU', bf16 / residual / remapped outputs -- are compiled out: the fit's GEMMs are small and latency bound.
template <bool FIT = false>
__device__ __forceinline__ float epi_pre(const GemmEpi& e, int m, int n, float acc) {
  float v = acc;
  if (e.bias) v += __ldg(e.bias + n);
  if (!FIT && e.act == ACT_GELU) v = gelu_erf(v);
  else if (e.act == ACT_RELU) v = fmaxf(v, 0.0f);
  if constexpr (!FIT) {
    if (e.mask) {
      float h = __bfloat162float(e.mask[(size_t)m * e.ldmask + n]);
      v = e.mask_mode == 1 ? v * gelu_grad(h) : (h > 0.0f ? v : 0.0f);
    }
  }
  if (e.mask_f32) v = e.mask_f32[(size_t)m * e.ldmask + n] > 0.0f ? v : 0.0f;
  return v * e.alpha;
}

__device__ __forceinline__ size_t epi_out_row(const GemmEpi& e, int m) {
  if (e.out_mode == OUT_F32_REMAP) {
    int g = m / e.rows_per_group;
    int p = m - g * e.rows_per_group;
    return (size_t)g * e.group_stride + e.row_offset + p;
  }
  return (size_t)m;
}

// bf16 copy of 4 consecutive pre-LayerScale values (OUT_F32_RESID with a branch buffer)
__device__ __forceinline__ void store_branch4(const GemmEpi& e, int m, int n, float4 v) {
  uint2 p;
  p.x = pack_bf16x2(v.x, v.y);
  p.y = pack_bf16x2(v.z, v.w);
  *reinterpret_cast<uint2*>(e.branch + (size_t)m * e.ld_branch + n) = p;
}

// scalar post-stage (SIMT debug path and ragged tails)
template <bool FIT = false>
__device__ __forceinline__ void epi_post1(const GemmEpi& e, int m, int n, float v) {
  size_t row = FIT ? (size_t)m : epi_out_row(e, m);
  if constexpr (FIT) {
    if (e.out_mode != OUT_F32 && e.out_mode != OUT_F32_ATOMIC && e.out_mode != OUT_F32_SPLIT) return;
  }
  switch (e.out_mode) {
    case OUT_BF16:
      reinterpret_cast<__nv_bfloat16*>(e.out)[row * e.ldo + n] = __float2bfloat16_rn(v);
      break;
    case OUT_F32:
      reinterpret_cast<float*>(e.out)[row * e.ldo + n] = v;
      break;
    case OUT_F32_ATOMIC:
      if (e.last_col_out && n == e.last_col_n) atomicAdd(e.last_col_out + m, v);
      else atomicAdd(reinterpret_cast<float*>(e.out) + row * e.ldo + n, v);
      break;
    case OUT_F32_RESID: {
      float* o = reinterpret_cast<float*>(e.out) + row * e.ldo + n;
      float g = e.gamma ? __ldg(e.gamma + n) : 1.0f;
      *o = fmaf(g, v, *o);
      if (e.branch) e.branch[(size_t)m * e.ld_branch + n] = __float2bfloat16_rn(v);
    } break;
    case OUT_F32_REMAP: {
      int p = m % e.rows_per_group;
      float a = e.addend ? __ldg(e.addend + (size_t)p * e.ldo + n) : 0.0f;
      reinterpret_cast<float*>(e.out)[row * e.ldo + n] = v + a;
    } break;
    case OUT_F32_SPLIT: {
      float* o = reinterpret_cast<float*>(e.out) + row * e.ldo + n;
      const float hi = tf32_hi(v);
      o[0] = hi;
      o[e.out_plane] = v - hi;
    } break;
  }
}

// vector post-stage: 4 consecutive columns, n % 4 == 0, ldo % 4 == 0, all in range
template <bool FIT = false>
__device__ __forceinline__ void epi_post4(const GemmEpi& e, int m, int n, float4 v) {
  if constexpr (FIT) {   // the three output forms of the fit, nothing else
    float* o = reinterpret_cast<float*>(e.out) + (size_t)m * e.ldo + n;
    if (e.out_mode == OUT_F32_SPLIT) {
      const float4 hi = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
      *reinterpret_cast<float4*>(o) = hi;
      *reinterpret_cast<float4*>(o + e.out_plane) = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
    } else if (e.out_mode == OUT_F32_ATOMIC) {
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                   : "memory");
    } else {
      *reinterpret_cast<float4*>(o) = v;
    }
    return;
  }
  size_t row = epi_out_row(e, m);
  switch (e.out_mode) {
    case OUT_BF16: {
      uint2 p;
      p.x = pack_bf16x2(v.x, v.y);
      p.y = pack_bf16x2(v.z, v.w);
      *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(e.out) + row * e.ldo + n) = p;
    } break;
    case OUT_F32:
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + row * e.ldo + n) = v;
      break;
    case OUT_F32_ATOMIC: {
      float* o = reinterpret_cast<float*>(e.out) + row * e.ldo + n;
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
                   : "memory");
    } break;
    case OUT_F32_RESID: {
      float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + row * e.ldo + n);
      float4 x = *o;
      float4 g = e.gamma ? __ldg(reinterpret_cast<const float4*>(e.gamma + n)) : make_float4(1.f, 1.f, 1.f, 1.f);
      x.x = fmaf(g.x, v.x, x.x);
      x.y = fmaf(g.y, v.y, x.y);
      x.z = fmaf(g.z, v.z, x.z);
      x.w = fmaf(g.w, v.w, x.w);
      *o = x;
      if (e.branch) store_branch4(e, m, n, v);
    } break;
    case OUT_F32_REMAP: {
      int p = m % e.rows_per_group;
      float4 a = e.addend ? __ldg(reinterpret_cast<const float4*>(e.addend + (size_t)p * e.ldo + n))
                          : make_float4(0.f, 0.f, 0.f, 0.f);
      v.x += a.x;
      v.y += a.y;
      v.z += a.z;
      v.w += a.w;
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + row * e.ldo + n) = v;
    } break;
    case OUT_F32_SPLIT: {
      float* o = reinterpret_cast<float*>(e.out) + row * e.ldo + n;
      const float4 hi = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
      *reinterpret_cast<float4*>(o) = hi;
      *reinterpret_cast<float4*>(o + e.out_plane) = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
    } break;
  }
}

// dtype: TMAP_BF16 (bf16 operands) or TMAP_F32 (TF32 products of fp32 operands; K-major only unless x3).
// lda / ldb: row pitch in elements of the stored matrix ([M,K] / [N,K], or [K,M] / [K,N] for MN-major operands).
// Runs the kernels debug_impl() selects.
int launch_gemm_tn(const void* A, int lda, const void* B, int ldb, TmapDtype dtype, const GemmShape& shape,
                   const GemmEpi& epi, cudaStream_t stream);

// out [M, N] (row pitch ldo) = the `splits` fp32 planes of an OUT_F32_PLANES GEMM summed in split order
int launch_splitk_planes_sum(const float* planes, int splits, size_t plane, int M, int N, int ldo, float* out,
                             cudaStream_t st);
int gemm_prepare();

}  // namespace dvt
