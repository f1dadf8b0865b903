// TN GEMM on Hopper tensor cores: C[M,N] = A[M,K] * B[N,K]^T with fused epilogues.
//
// bf16 and TF32 products (gemm_wgmma_kernel): one 128 x 128 output tile per CTA, 9 warps:
//   warps 0-7   two consumer warpgroups, 64 rows each: wgmma m64n128 (k16 bf16 / k8 tf32) straight from the swizzled TMA
//               tiles (bf16 operands K-major or MN-major, TF32 K-major), fp32 accumulators in registers
//   warp 8      TMA producer (A: 128 x 128B, B: 128 x 128B per stage, SWIZZLE_128B, 3-stage mbarrier ring)
//   The accumulators are then staged through shared memory (the drained operand ring) and the eight consumer warps run
//   the fused epilogue on 32 x 32 chunks in a coalesced layout.  Three stages (96 KB) keep two CTAs resident per SM, so
//   one CTA's epilogue overlaps the other's main loop.
// 3xTF32 products (fp32 hi/lo operand planes):
//   both operands K-major -- every product of the stage-1 fit: the forward linears and data gradients, and the weight
//   gradients dY^T [X | 1], which read transposed copies of dY and X written by their producers (GemmEpi::out_t):
//   gemm_wgmma_x3_kernel, 128 x 64 tiles of wgmma m64n64k8 TF32, two CTAs per SM
//   an MN-major operand (dvt_gemm_f32x3 only): gemm_x3_kernel, 128 x 64 tiles, 8 warps of mma.sync m16n8k8 TF32 with
//   fragments read from the swizzled TMA tiles -- wgmma's TF32 form takes K-major operands only.
// K tails, M tails and N tails are handled by TMA zero-fill plus masking in the epilogue.
//
// Used for: patch-embed, QKV, attention out-proj, MLP fc1/fc2 (reference: timm VisionTransformer reached from
// dvt/models/vit_wrapper.py:136-143) and for the field / residual MLP forward+backward of the stage-1 fit
// (reference: dvt/models/neural_feature_field.py:40-44, dvt/models/offline_denoiser.py:40-46).
#include "gemm.cuh"

#include <algorithm>

namespace dvt {

namespace {

constexpr int BM = 128;
constexpr int KB_BYTES = 128;  // bytes of K per pipeline stage row (= one 128B swizzle atom)

// wgmma kernel
constexpr int WG_BN = 128;
constexpr int WG_STAGES = 3;
constexpr int WG_THREADS = 288;                      // 2 consumer warpgroups + 1 producer warp
constexpr int WG_STAGE_BYTES = (BM + WG_BN) * KB_BYTES;
constexpr int WG_OFF_BAR = WG_STAGES * WG_STAGE_BYTES;
constexpr int WG_SMEM = WG_OFF_BAR + 2 * WG_STAGES * 8 + 1024;  // + alignment slack
constexpr int EPI_PITCH = WG_BN + 8;                 // floats per staged accumulator row (16B aligned, conflict-free)
static_assert(BM * EPI_PITCH * 4 <= WG_OFF_BAR, "staged accumulators must fit in the operand ring");
static_assert(2 * WG_SMEM <= 227 * 1024, "two CTAs per SM");

// 3xTF32 kernel
constexpr int X3_STAGES = 3;
constexpr int X3_THREADS = 256;
template <int BN>
struct X3Smem {
  static constexpr int A_BYTES = 2 * BM * KB_BYTES;  // hi plane then lo plane (K-major) / 32-column atoms (MN-major)
  static constexpr int B_BYTES = 2 * BN * KB_BYTES;
  static constexpr int STAGE = A_BYTES + B_BYTES;
  static constexpr int OFF_BAR = X3_STAGES * STAGE;
  static constexpr int PITCH = BN + 8;
  static constexpr int TOTAL = OFF_BAR + X3_STAGES * 8 + 1024;
  static_assert(BM * PITCH * 4 <= OFF_BAR, "staged accumulators must fit in the operand ring");
};

// A never-taken branch at the entry of the wgmma and 3xTF32 kernels (GemmEpi::entry_guard is always null).  It does nothing
// at run time, but nvcc 12.9 allocates registers for these kernels better with it.  Without it (measured when it was
// added) the gemm_x3_kernel instantiations took up to 24 more registers, the gemm_wgmma_kernel ones went from 90 to 92, and
// gemm_wgmma_swiglu_bwd_kernel spilled 4 bytes.  An empty asm statement or moving tile_of() does not have the same effect.
__device__ __forceinline__ void gemm_entry_guard(const GemmEpi& e) {
  if (threadIdx.x == 0 && e.entry_guard && blockIdx.x == 0) e.entry_guard[0] = 0;
}

template <bool FIT>
__device__ __forceinline__ void epi_scalar_tail(const GemmEpi& e, const GemmShape& s, float* scr, int pitch, int lane,
                                                int m0, int n, bool has_k) {
#pragma unroll 1
  for (int jj = 0; jj < 8; ++jj) {
    const int i = (lane >> 3) + 4 * jj;
    const int m = m0 + 4 * jj;
    if (m >= s.M) continue;
#pragma unroll 1
    for (int q = 0; q < 4; ++q) {
      if (n + q >= s.N) break;
      float* x = scr + i * pitch + (lane & 7) * 4 + q;
      const float v = epi_pre<FIT>(e, m, n + q, has_k ? *x : 0.0f);
      epi_post1<FIT>(e, m, n + q, v);
      if (FIT && e.out_t) *x = v;  // read back by epi_store_t
    }
  }
}

// One 32-row x 32-column chunk of an accumulator tile staged in shared memory (`scr`: the chunk's first element, rows
// `pitch` floats apart), with the fused epilogue in the coalesced layout (each lane: 4 consecutive columns of 8 rows).
// FIT with GemmEpi::out_t: the epilogue's values replace the accumulators in `scr`, for epi_store_t.
// m0: global row of this lane's first row (chunk row base + lane / 8); n_base: global column of the chunk.  Everything
// that depends on the column (bias, LayerScale, ...) is loaded once per chunk as a float4.
template <bool FIT = false>
__device__ __forceinline__ void epi_chunk(const GemmEpi& e, const GemmShape& s, float* scr, int pitch, int lane,
                                          int n_base, int m0, bool has_k) {
  const int col4 = (lane & 7) * 4;
  const int n = n_base + col4;
  if (n + 3 < s.N) {
    // ---------------- vector path ----------------
    float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (e.bias) b4 = __ldg(reinterpret_cast<const float4*>(e.bias + n));
    float4 g4 = make_float4(1.f, 1.f, 1.f, 1.f);
    if (e.out_mode == OUT_F32_RESID && e.gamma) g4 = __ldg(reinterpret_cast<const float4*>(e.gamma + n));
    float4 xin[8];
    if (!FIT && e.out_mode == OUT_F32_RESID) {  // issue all residual loads before any store (memory-level parallelism)
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int m = m0 + 4 * jj;
        if (m < s.M) xin[jj] = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(e.out) + (size_t)m * e.ldo + n);
      }
    }
    const bool plain = e.mask == nullptr && e.mask_f32 == nullptr && e.alpha == 1.0f && has_k;
    if (!FIT && plain && e.out_mode == OUT_BF16) {
      // ---- fast path: bias (+ GELU / ReLU) -> bf16.  The activation is chosen ONCE per chunk, the row loop is
      // branch-free (QKV and fc1+GELU, the two largest epilogues of the ViT forward).
      __nv_bfloat16* outp = reinterpret_cast<__nv_bfloat16*>(e.out);
      if (e.act == ACT_GELU) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int m = m0 + 4 * jj;
          float4 x = *reinterpret_cast<const float4*>(scr + ((lane >> 3) + 4 * jj) * pitch + col4);
          uint2 pk;
          const float2 g01 = gelu_erf2(fadd2(make_float2(x.x, x.y), make_float2(b4.x, b4.y)));
          const float2 g23 = gelu_erf2(fadd2(make_float2(x.z, x.w), make_float2(b4.z, b4.w)));
          pk.x = pack_bf16x2(g01.x, g01.y);
          pk.y = pack_bf16x2(g23.x, g23.y);
          if (m < s.M) *reinterpret_cast<uint2*>(outp + (size_t)m * e.ldo + n) = pk;
        }
      } else if (e.act == ACT_RELU) {
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int m = m0 + 4 * jj;
          float4 x = *reinterpret_cast<const float4*>(scr + ((lane >> 3) + 4 * jj) * pitch + col4);
          uint2 pk;
          pk.x = pack_bf16x2(fmaxf(x.x + b4.x, 0.0f), fmaxf(x.y + b4.y, 0.0f));
          pk.y = pack_bf16x2(fmaxf(x.z + b4.z, 0.0f), fmaxf(x.w + b4.w, 0.0f));
          if (m < s.M) *reinterpret_cast<uint2*>(outp + (size_t)m * e.ldo + n) = pk;
        }
      } else {   // bias only (QKV): two FADD2 and two packs per four outputs
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int m = m0 + 4 * jj;
          float4 x = *reinterpret_cast<const float4*>(scr + ((lane >> 3) + 4 * jj) * pitch + col4);
          const float2 v01 = fadd2(make_float2(x.x, x.y), make_float2(b4.x, b4.y));
          const float2 v23 = fadd2(make_float2(x.z, x.w), make_float2(b4.z, b4.w));
          uint2 pk;
          pk.x = pack_bf16x2(v01.x, v01.y);
          pk.y = pack_bf16x2(v23.x, v23.y);
          if (m < s.M) *reinterpret_cast<uint2*>(outp + (size_t)m * e.ldo + n) = pk;
        }
      }
    } else if (!FIT && plain && e.out_mode == OUT_F32_RESID && e.act == ACT_NONE) {
      // ---- fast path: x += gamma * (acc + bias)  (attention out-proj, fc2) ----
      float* outp = reinterpret_cast<float*>(e.out);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const int m = m0 + 4 * jj;
        const float4 x = *reinterpret_cast<const float4*>(scr + ((lane >> 3) + 4 * jj) * pitch + col4);
        const float2 o01 = ffma2(make_float2(g4.x, g4.y), fadd2(make_float2(x.x, x.y), make_float2(b4.x, b4.y)),
                                 make_float2(xin[jj].x, xin[jj].y));
        const float2 o23 = ffma2(make_float2(g4.z, g4.w), fadd2(make_float2(x.z, x.w), make_float2(b4.z, b4.w)),
                                 make_float2(xin[jj].z, xin[jj].w));
        if (m < s.M) {
          *reinterpret_cast<float4*>(outp + (size_t)m * e.ldo + n) = make_float4(o01.x, o01.y, o23.x, o23.y);
          if (e.branch) {
            const float2 v01 = fadd2(make_float2(x.x, x.y), make_float2(b4.x, b4.y));
            const float2 v23 = fadd2(make_float2(x.z, x.w), make_float2(b4.z, b4.w));
            store_branch4(e, m, n, make_float4(v01.x, v01.y, v23.x, v23.y));
          }
        }
      }
    } else {
      // ---- generic path (fit epilogues: masks, split planes, atomics, remap) ----
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
      const int i = (lane >> 3) + 4 * jj;
      const int m = m0 + 4 * jj;
      float4 x = *reinterpret_cast<const float4*>(scr + i * pitch + col4);
      if (m >= s.M) continue;
      if (!has_k) x = make_float4(0.f, 0.f, 0.f, 0.f);
      x.x += b4.x; x.y += b4.y; x.z += b4.z; x.w += b4.w;
      if (!FIT && e.act == ACT_GELU) {
        x.x = gelu_erf(x.x); x.y = gelu_erf(x.y); x.z = gelu_erf(x.z); x.w = gelu_erf(x.w);
      } else if (e.act == ACT_RELU) {
        x.x = fmaxf(x.x, 0.f); x.y = fmaxf(x.y, 0.f); x.z = fmaxf(x.z, 0.f); x.w = fmaxf(x.w, 0.f);
      }
      if (e.mask_f32) {
        const float4 h = *reinterpret_cast<const float4*>(e.mask_f32 + (size_t)m * e.ldmask + n);
        x.x = h.x > 0.f ? x.x : 0.f; x.y = h.y > 0.f ? x.y : 0.f; x.z = h.z > 0.f ? x.z : 0.f; x.w = h.w > 0.f ? x.w : 0.f;
      } else if (!FIT && e.mask) {
        const uint2 hb = *reinterpret_cast<const uint2*>(e.mask + (size_t)m * e.ldmask + n);
        const __nv_bfloat162 h01 = *reinterpret_cast<const __nv_bfloat162*>(&hb.x);
        const __nv_bfloat162 h23 = *reinterpret_cast<const __nv_bfloat162*>(&hb.y);
        if (e.mask_mode == 1) {  // GELU backward: the mask tensor is the forward pre-activation
          x.x *= gelu_grad(__low2float(h01)); x.y *= gelu_grad(__high2float(h01));
          x.z *= gelu_grad(__low2float(h23)); x.w *= gelu_grad(__high2float(h23));
        } else {
          x.x = __low2float(h01) > 0.f ? x.x : 0.f; x.y = __high2float(h01) > 0.f ? x.y : 0.f;
          x.z = __low2float(h23) > 0.f ? x.z : 0.f; x.w = __high2float(h23) > 0.f ? x.w : 0.f;
        }
      }
      if (e.alpha != 1.0f) { x.x *= e.alpha; x.y *= e.alpha; x.z *= e.alpha; x.w *= e.alpha; }
      if (FIT && e.out_t) *reinterpret_cast<float4*>(scr + i * pitch + col4) = x;
      if (!FIT && e.out_mode == OUT_F32_RESID) {
        float4 o = xin[jj];
        o.x = fmaf(g4.x, x.x, o.x); o.y = fmaf(g4.y, x.y, o.y); o.z = fmaf(g4.z, x.z, o.z); o.w = fmaf(g4.w, x.w, o.w);
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(e.out) + (size_t)m * e.ldo + n) = o;
        if (e.branch) store_branch4(e, m, n, x);
      } else {
        epi_post4<FIT>(e, m, n, x);
      }
    }
    }
  } else {
    // ---------------- ragged N tail: scalar path ----------------
    epi_scalar_tail<FIT>(e, s, scr, pitch, lane, m0, n, has_k);
  }
  }

// SwiGLU backward (mask_mode 2, dvt_gemm_bf16_dgrad_swiglu).  The product is dh = dY . W2 [M, Hh] with Hh = s.N; e.mask is
// the saved fc1 output hpre [M, 2 Hh] = [g | u] (timm SwiGLUPacked chunk order), e.out receives dhpre bf16 [M, 2 Hh]:
//   dhpre[m, n] = dh * u * silu'(g),   dhpre[m, n + Hh] = dh * silu(g).
// silu(g) = g / (1 + exp(-g)) is the expression of swiglu_kernel (the forward); silu'(g) = s + silu(g) (1 - s) with
// s = 1 / (1 + exp(-g)) stays finite where exp(-g) overflows (s = 0, silu(g) = -0).  Returns (dg, du).
__device__ __forceinline__ float2 swiglu_bwd(float dh, float g, float u) {
  const float den = 1.0f + __expf(-g);
  const float s = 1.0f / den;
  const float sl = g / den;
  return make_float2(dh * u * fmaf(sl, 1.0f - s, s), dh * sl);
}

__device__ __forceinline__ void swiglu_bwd_store1(const GemmEpi& e, int m, int n, int Hh, float dh) {
  const size_t ri = (size_t)m * e.ldmask, ro = (size_t)m * e.ldo;
  const float2 d = swiglu_bwd(dh, __bfloat162float(e.mask[ri + n]), __bfloat162float(e.mask[ri + n + Hh]));
  __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(e.out);
  o[ro + n] = __float2bfloat16_rn(d.x);
  o[ro + n + Hh] = __float2bfloat16_rn(d.y);
}

// epi_chunk of the SwiGLU backward: each lane reads 4 consecutive g and the 4 matching u of 8 rows (all loads issued before
// any use) and stores 4 columns in each half, both coalesced.  An Hh that is not a multiple of 4 (possible with a padded
// W2) takes the scalar path everywhere: the second half would not be 8-byte aligned.
__device__ __forceinline__ void epi_chunk_swiglu_bwd(const GemmEpi& e, const GemmShape& s, const float* scr, int pitch,
                                                     int lane, int n_base, int m0, bool has_k) {
  const int col4 = (lane & 7) * 4;
  const int n = n_base + col4;
  const int Hh = s.N;
  if (n >= Hh) return;
  if ((Hh & 3) == 0) {
    uint2 gv[8], uv[8];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int m = m0 + 4 * jj;
      if (m < s.M) {
        const __nv_bfloat16* h = e.mask + (size_t)m * e.ldmask + n;
        gv[jj] = *reinterpret_cast<const uint2*>(h);
        uv[jj] = *reinterpret_cast<const uint2*>(h + Hh);
      }
    }
    __nv_bfloat16* outp = reinterpret_cast<__nv_bfloat16*>(e.out);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      const int m = m0 + 4 * jj;
      if (m >= s.M) continue;
      float4 x = *reinterpret_cast<const float4*>(scr + ((lane >> 3) + 4 * jj) * pitch + col4);
      if (!has_k) x = make_float4(0.f, 0.f, 0.f, 0.f);
      const float2 g01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&gv[jj].x));
      const float2 g23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&gv[jj].y));
      const float2 u01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&uv[jj].x));
      const float2 u23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&uv[jj].y));
      const float2 d0 = swiglu_bwd(x.x, g01.x, u01.x), d1 = swiglu_bwd(x.y, g01.y, u01.y);
      const float2 d2 = swiglu_bwd(x.z, g23.x, u23.x), d3 = swiglu_bwd(x.w, g23.y, u23.y);
      __nv_bfloat16* o = outp + (size_t)m * e.ldo + n;
      *reinterpret_cast<uint2*>(o) = make_uint2(pack_bf16x2(d0.x, d1.x), pack_bf16x2(d2.x, d3.x));
      *reinterpret_cast<uint2*>(o + Hh) = make_uint2(pack_bf16x2(d0.y, d1.y), pack_bf16x2(d2.y, d3.y));
    }
  } else {
#pragma unroll 1
    for (int jj = 0; jj < 8; ++jj) {
      const int m = m0 + 4 * jj;
      if (m >= s.M) continue;
#pragma unroll 1
      for (int q = 0; q < 4 && n + q < Hh; ++q) {
        const float x = scr[((lane >> 3) + 4 * jj) * pitch + col4 + q];
        swiglu_bwd_store1(e, m, n + q, Hh, has_k ? x : 0.0f);
      }
    }
  }
}

// epi_chunk of the QKV projection with the 2-D RoPE (GemmEpi::rope): a q / k chunk (32 columns, one half of a 64-wide head)
// reads the matching 32 columns of the other half from the staged tile -- the 128-wide tile holds whole heads -- so the
// rotation acts on the fp32 accumulators before the one bf16 store.  Each lane: 4 consecutive columns d of 8 rows, the
// 4 partners d +- 32, and per patch row one float4 of cos and one of sin.
__device__ __forceinline__ void epi_chunk_rope(const GemmEpi& e, const GemmShape& s, const float* scr, int pitch, int lane,
                                               int n_base, int m0) {
  const int col4 = (lane & 7) * 4;
  const int n = n_base + col4;
  const bool upper = (n_base & 32) != 0;   // second half of the head: out = v cos + v[d - 32] sin
  const int dp = upper ? -32 : 32;
  float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f), bp = b4;
  if (e.bias) {
    b4 = __ldg(reinterpret_cast<const float4*>(e.bias + n));
    bp = __ldg(reinterpret_cast<const float4*>(e.bias + n + dp));
  }
  const float sg = upper ? 1.0f : -1.0f;
  __nv_bfloat16* outp = reinterpret_cast<__nv_bfloat16*>(e.out);
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
    const int m = m0 + 4 * jj;
    if (m >= s.M) continue;
    const float* r = scr + ((lane >> 3) + 4 * jj) * pitch + col4;
    float4 x = *reinterpret_cast<const float4*>(r);
    x.x += b4.x; x.y += b4.y; x.z += b4.z; x.w += b4.w;
    const int t = m % e.rope_ntok;
    if (t >= e.rope_prefix) {
      float4 y = *reinterpret_cast<const float4*>(r + dp);
      y.x += bp.x; y.y += bp.y; y.z += bp.z; y.w += bp.w;
      const float* cs = e.rope + (size_t)(t - e.rope_prefix) * 64 + (col4 & 31);
      const float4 c = __ldg(reinterpret_cast<const float4*>(cs));
      const float4 sn = __ldg(reinterpret_cast<const float4*>(cs + 32));
      x.x = x.x * c.x + sg * (y.x * sn.x);
      x.y = x.y * c.y + sg * (y.y * sn.y);
      x.z = x.z * c.z + sg * (y.z * sn.z);
      x.w = x.w * c.w + sg * (y.w * sn.w);
    }
    uint2 pk;
    pk.x = pack_bf16x2(x.x, x.y);
    pk.y = pack_bf16x2(x.z, x.w);
    *reinterpret_cast<uint2*>(outp + (size_t)m * e.ldo + n) = pk;
  }
}


// Tile t of a launch: (split, tile_n, tile_m), split fastest.
struct TileIdx {
  int tm, tn, kb0, kb1, kb_total;
};
__device__ __forceinline__ TileIdx tile_of(const GemmShape& s, int bn, int bk) {
  TileIdx r;
  const int tiles_n = (s.N + bn - 1) / bn;
  const int t = blockIdx.x;
  const int split = t % s.splits;
  const int mn = t / s.splits;
  r.tn = mn % tiles_n;
  r.tm = mn / tiles_n;
  r.kb_total = (s.K + bk - 1) / bk;
  const int per = (r.kb_total + s.splits - 1) / s.splits;
  r.kb0 = split * per;
  r.kb1 = min(r.kb_total, r.kb0 + per);
  return r;
}

// Epilogue of a tile whose fp32 accumulators sit in shared memory ([BM][pitch]): warp w of `nwarps` takes the 32 x 32
// chunks w, w + nwarps, ...  GLU: the SwiGLU-backward epilogue (epi_chunk_swiglu_bwd) instead of epi_chunk; ROPE: the q / k
// chunks take epi_chunk_rope.  Compile-time switches, so that no other instantiation carries their code.
template <bool FIT, int BN, bool GLU = false, bool ROPE = false>
__device__ __forceinline__ void epi_tile(const GemmEpi& e, const GemmShape& s, float* tile, int pitch, int warp,
                                         int nwarps, int lane, int tm, int tn, bool has_k) {
#pragma unroll 1
  for (int c = warp; c < (BM / 32) * (BN / 32); c += nwarps) {
    const int rb = c / (BN / 32), cb = c % (BN / 32);
    const int n_base = tn * BN + cb * 32;
    if (n_base >= s.N || tm * BM + rb * 32 >= s.M) continue;  // whole chunk out of range (warp-uniform)
    if (ROPE && n_base < e.rope_cols)
      epi_chunk_rope(e, s, tile + rb * 32 * pitch + cb * 32, pitch, lane, n_base, tm * BM + rb * 32 + (lane >> 3));
    else if constexpr (GLU)
      epi_chunk_swiglu_bwd(e, s, tile + rb * 32 * pitch + cb * 32, pitch, lane, n_base, tm * BM + rb * 32 + (lane >> 3), has_k);
    else
      epi_chunk<FIT>(e, s, tile + rb * 32 * pitch + cb * 32, pitch, lane, n_base, tm * BM + rb * 32 + (lane >> 3), has_k);
  }
}

// Body of the wgmma kernels (below): gemm_wgmma_kernel<TF32, A_MN, B_MN> with the general epilogue,
// gemm_wgmma_swiglu_bwd_kernel (bf16, B MN-major) with the SwiGLU-backward one, gemm_wgmma_planes_kernel (bf16, both
// MN-major; PLANES: split k stores its partial tile into plane k of e.out, the OUT_F32_PLANES mode) and
// gemm_wgmma_rope_kernel (bf16, both K-major; ROPE: the QKV projection with the 2-D RoPE epilogue).
template <bool TF32, bool A_MN, bool B_MN, bool GLU, bool PLANES = false, bool ROPE = false>
__device__ __forceinline__ void wgmma_gemm_body(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmShape& s,
                                                const GemmEpi& e) {
  static_assert(!(TF32 && (A_MN || B_MN)), "TF32 wgmma operands are K-major only");
  constexpr int BK = KB_BYTES / (TF32 ? 4 : 2);  // elements of K per stage
  constexpr int A_BYTES = BM * KB_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + WG_OFF_BAR);
  uint64_t* empty = full + WG_STAGES;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  gemm_entry_guard(e);
  const TileIdx ti = tile_of(s, WG_BN, BK);

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < WG_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  // PDL: everything above overlapped the tail of the previous kernel; its results are needed from here on
  pdl_wait();
  pdl_trigger();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      for (int kb = ti.kb0, it = 0; kb < ti.kb1; ++kb, ++it) {
        const int st = it % WG_STAGES;
        mbar_wait_relaxed(&empty[st], ((it / WG_STAGES) & 1) ^ 1, 1);
        uint8_t* sA = smem + st * WG_STAGE_BYTES;
        uint8_t* sB = sA + A_BYTES;
        mbar_expect_tx(&full[st], WG_STAGE_BYTES);
        if (A_MN) {  // stored [K, M]: boxes of 64 (M, contiguous) x BK (K rows) = one MN-major swizzle-atom column each
#pragma unroll
          for (int a = 0; a < BM / 64; ++a) tma_load_2d(sA + a * (BK * 128), &tmA, &full[st], ti.tm * BM + a * 64, kb * BK);
        } else {
          tma_load_2d(sA, &tmA, &full[st], kb * BK, ti.tm * BM);
        }
        if (B_MN) {
#pragma unroll
          for (int a = 0; a < WG_BN / 64; ++a) tma_load_2d(sB + a * (BK * 128), &tmB, &full[st], ti.tn * WG_BN + a * 64, kb * BK);
        } else {
          tma_load_2d(sB, &tmB, &full[st], kb * BK, ti.tn * WG_BN);
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;  // rows [64 wg, 64 wg + 64) of the tile
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  reg_fence(acc);
  for (int kb = ti.kb0, it = 0; kb < ti.kb1; ++kb, ++it) {
    const int st = it % WG_STAGES;
    mbar_wait(&full[st], (it / WG_STAGES) & 1, 3);
    const uint32_t a_base = smem_u32(smem + st * WG_STAGE_BYTES), b_base = a_base + A_BYTES;
    // K-major: rows of 128 B, K advances 32 B per MMA.  MN-major: [64-wide atoms, BK * 128 B apart][BK k-rows of 128 B];
    // K advances 16 rows = 2048 B per MMA.
    const uint64_t da = A_MN ? make_wgmma_desc(a_base + wg * (BK * 128), BK * 128, 1024) : make_wgmma_desc(a_base + wg * 64 * 128, 0, 1024);
    const uint64_t db = make_wgmma_desc(b_base, B_MN ? BK * 128 : 0, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t adv_a = (uint64_t)((A_MN ? k * 2048 : k * 32) >> 4);
      const uint64_t adv_b = (uint64_t)((B_MN ? k * 2048 : k * 32) >> 4);
      if constexpr (TF32) wgmma_128_tf32(acc, da + adv_a, db + adv_b);
      else wgmma_128_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da + adv_a, db + adv_b);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the MMAs of the previous stage have completed: release its slot
    reg_fence(acc);
    if (it > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[(it - 1) % WG_STAGES]);
    }
  }
  wgmma_wait<0>();
  reg_fence(acc);

  // ---- stage the accumulators in the drained operand ring, then the fused epilogue ----
  named_bar(1, 256);  // both warpgroups are done reading operands
  float* tile = reinterpret_cast<float*>(smem);
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      *reinterpret_cast<float2*>(tile + r0 * EPI_PITCH + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(tile + (r0 + 8) * EPI_PITCH + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  named_bar(1, 256);
  if constexpr (PLANES) {  // plain fp32 stores into this split's plane
    GemmEpi ep = e;
    ep.out_mode = OUT_F32;
    ep.out = reinterpret_cast<float*>(e.out) + (size_t)(blockIdx.x % s.splits) * e.out_plane;
    epi_tile<false, WG_BN, false>(ep, s, tile, EPI_PITCH, warp, 8, lane, ti.tm, ti.tn, ti.kb0 < ti.kb_total);
  } else {
    epi_tile<false, WG_BN, GLU, ROPE>(e, s, tile, EPI_PITCH, warp, 8, lane, ti.tm, ti.tn, ti.kb0 < ti.kb_total);
  }
}

template <bool TF32, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(WG_THREADS, 2)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmShape s, GemmEpi e) {
  wgmma_gemm_body<TF32, A_MN, B_MN, false>(tmA, tmB, s, e);
}

// fc2 data gradient of a SwiGLU MLP: dY [M, C] (K-major) . W2 stored [C, Hh] (MN-major), SwiGLU backward in the epilogue
__global__ void __launch_bounds__(WG_THREADS, 2)
gemm_wgmma_swiglu_bwd_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmShape s,
                             GemmEpi e) {
  wgmma_gemm_body<false, false, true, true>(tmA, tmB, s, e);
}

// Split-K weight gradient without atomics (OUT_F32_PLANES): A and B MN-major (activations in their [rows, features] storage)
__global__ void __launch_bounds__(WG_THREADS, 2)
gemm_wgmma_planes_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmShape s,
                         GemmEpi e) {
  wgmma_gemm_body<false, true, true, false, true>(tmA, tmB, s, e);
}

// QKV projection of a RoPE ViT (DINOv3): x [M, C] . Wqkv [3C, C]^T + bias, q and k of the patch rows rotated in the epilogue
__global__ void __launch_bounds__(WG_THREADS, 2)
gemm_wgmma_rope_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmShape s,
                       GemmEpi e) {
  wgmma_gemm_body<false, false, false, false, false, true>(tmA, tmB, s, e);
}

// ----------------------------------------------------------------------------------------------------
// 3xTF32 ("x3"): fp32-accurate products of fp32 operands stored as hi / lo planes.  Per stage a 128 x 32 slab of A and a
// BN x 32 slab of B, both planes, through TMA with 128-byte swizzle:
//   K-major operand   [plane][rows][32 fp32]                    (one 3-D box)
//   MN-major operand  [32-wide atoms][plane][32 k-rows][32 fp32] (one 3-D box per atom)
// 8 warps in a 4 (M) x 2 (N) grid, each 32 x BN/2 of the tile.
// ----------------------------------------------------------------------------------------------------
template <int ROWS, bool MN>
__device__ __forceinline__ uint32_t x3_ld(const uint8_t* base, int r, int k, int plane) {
  uint32_t off;
  if (MN) off = (r >> 5) * 8192 + plane * 4096 + k * 128 + ((((r & 31) >> 2) ^ (k & 7)) << 4) + (r & 3) * 4;
  else off = plane * (ROWS * 128) + r * 128 + (((k >> 2) ^ (r & 7)) << 4) + (k & 3) * 4;
  return *reinterpret_cast<const uint32_t*>(base + off);
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

template <int BN, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(X3_THREADS, 1)
gemm_x3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmShape s, GemmEpi e) {
  using L = X3Smem<BN>;
  constexpr int BK = 32;
  constexpr int WN = BN / 2;   // columns per warp
  constexpr int NT = WN / 8;   // n8 sub-tiles per warp
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;
  gemm_entry_guard(e);
  const TileIdx ti = tile_of(s, BN, BK);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < X3_STAGES; ++i) mbar_init(&full[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  auto issue = [&](int kb, int st) {
    uint8_t* sA = smem + st * L::STAGE;
    uint8_t* sB = sA + L::A_BYTES;
    mbar_expect_tx(&full[st], L::STAGE);
    if (A_MN) {
#pragma unroll
      for (int a = 0; a < BM / 32; ++a) tma_load_3d(sA + a * 8192, &tmA, &full[st], ti.tm * BM + a * 32, kb * BK, 0);
    } else {
      tma_load_3d(sA, &tmA, &full[st], kb * BK, ti.tm * BM, 0);
    }
    if (B_MN) {
#pragma unroll
      for (int a = 0; a < BN / 32; ++a) tma_load_3d(sB + a * 8192, &tmB, &full[st], ti.tn * BN + a * 32, kb * BK, 0);
    } else {
      tma_load_3d(sB, &tmB, &full[st], kb * BK, ti.tn * BN, 0);
    }
  };
  if (threadIdx.x == 0)
    for (int i = 0; i < X3_STAGES && ti.kb0 + i < ti.kb1; ++i) issue(ti.kb0 + i, i);

  float acc[2][NT][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < NT; ++ni)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[mi][ni][q] = 0.f;

  for (int kb = ti.kb0, it = 0; kb < ti.kb1; ++kb, ++it) {
    const int st = it % X3_STAGES;
    mbar_wait(&full[st], (it / X3_STAGES) & 1, 3);
    const uint8_t* sA = smem + st * L::STAGE;
    const uint8_t* sB = sA + L::A_BYTES;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 8) {
      uint32_t ah[2][4], al[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int r = wm * 32 + mi * 16 + g;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int rr = r + (q & 1) * 8, k = kk + t + (q >> 1) * 4;
          ah[mi][q] = x3_ld<BM, A_MN>(sA, rr, k, 0);
          al[mi][q] = x3_ld<BM, A_MN>(sA, rr, k, 1);
        }
      }
#pragma unroll
      for (int ni = 0; ni < NT; ++ni) {
        const int n = wn * WN + ni * 8 + g;
        uint32_t bh[2], bl[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          bh[q] = x3_ld<BN, B_MN>(sB, n, kk + t + 4 * q, 0);
          bl[q] = x3_ld<BN, B_MN>(sB, n, kk + t + 4 * q, 1);
        }
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          mma_tf32(acc[mi][ni], al[mi], bh);  // small terms first
          mma_tf32(acc[mi][ni], ah[mi], bl);
          mma_tf32(acc[mi][ni], ah[mi], bh);
        }
      }
    }
    __syncthreads();  // every warp is done with this slot
    if (threadIdx.x == 0 && kb + X3_STAGES < ti.kb1) issue(kb + X3_STAGES, st);
  }

  // ---- stage the accumulators in the drained operand ring, then the fused epilogue ----
  float* tile = reinterpret_cast<float*>(smem);
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < NT; ++ni) {
      const int r = wm * 32 + mi * 16 + g, c = wn * WN + ni * 8 + 2 * t;
      *reinterpret_cast<float2*>(tile + r * L::PITCH + c) = make_float2(acc[mi][ni][0], acc[mi][ni][1]);
      *reinterpret_cast<float2*>(tile + (r + 8) * L::PITCH + c) = make_float2(acc[mi][ni][2], acc[mi][ni][3]);
    }
  __syncthreads();
  // split-K with counters: split k of a tile adds its partial sums once splits 0 .. k-1 have added theirs (lower block
  // indices, scheduled first), so every element is summed in split order
  const bool serial = e.splitk_sem != nullptr && s.splits > 1;
  unsigned* sem = e.splitk_sem + blockIdx.x / s.splits;
  const unsigned split = blockIdx.x % s.splits;
  if (serial) {
    if (threadIdx.x == 0) {
      const long long t0 = clock64();
      while (ld_acquire_u32(sem) != split)
        if (clock64() - t0 > DVT_WATCHDOG_CYCLES) dev_fail(0x5E3u, split);
    }
    __syncthreads();
  }
  epi_tile<true, BN>(e, s, tile, L::PITCH, warp, 8, lane, ti.tm, ti.tn, ti.kb0 < ti.kb_total);
  if (serial) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) st_release_u32(sem, split + 1 == (unsigned)s.splits ? 0u : split + 1);
  }
}

// ----------------------------------------------------------------------------------------------------
// 3xTF32 on wgmma (gemm_wgmma_x3_kernel): both operands K-major hi / lo planes, 128 x 64 output tiles, 9 warps as in
// gemm_wgmma_kernel.  Per stage one 3-D TMA box per operand ([plane][rows][32 fp32], 128-byte swizzle: two ordinary
// K-major wgmma tiles, hi then lo).  Each k8 step issues A_lo.B_hi, A_hi.B_lo, A_hi.B_hi (the order of gemm_x3_kernel)
// into one fp32 accumulator.  Two stages (96 KB) keep two CTAs on an SM: the fit's GEMMs are 2048 rows by 128-768
// columns, 48-192 tiles, so one CTA's epilogue and ramp-up overlap the other's main loop.
// ----------------------------------------------------------------------------------------------------
constexpr int X3W_BN = 64;
constexpr int X3W_STAGES = 2;
constexpr int X3W_A_BYTES = 2 * BM * KB_BYTES;
constexpr int X3W_STAGE = X3W_A_BYTES + 2 * X3W_BN * KB_BYTES;
constexpr int X3W_OFF_BAR = X3W_STAGES * X3W_STAGE;
constexpr int X3W_PITCH = X3W_BN + 8;
constexpr int X3W_SMEM = X3W_OFF_BAR + 2 * X3W_STAGES * 8 + 1024;
static_assert(BM * X3W_PITCH * 4 <= X3W_OFF_BAR, "staged accumulators must fit in the operand ring");
static_assert(2 * (X3W_SMEM + 1024) <= 228 * 1024, "two CTAs per SM");

// GemmEpi::out_t of a tile whose epilogue values epi_tile has left in `tile` ([BM][pitch]): thread t of the 256 takes row
// t % 128 and half t / 128 of the 64 columns, so each store of a warp writes 32 consecutive m of one transposed row.
__device__ __forceinline__ void epi_store_t(const GemmEpi& e, const GemmShape& s, const float* tile, int pitch, int tm,
                                            int tn) {
  const int r = threadIdx.x & (BM - 1), m = tm * BM + r;
  if (m >= s.M) return;
  const int c0 = (threadIdx.x >> 7) * (X3W_BN / 2);
#pragma unroll 2
  for (int c = c0; c < c0 + X3W_BN / 2; c += 4) {
    const int n = tn * X3W_BN + c;
    if (n >= s.N) break;
    const float4 v4 = *reinterpret_cast<const float4*>(tile + r * pitch + c);
    const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (n + q >= s.N) break;
      const float hi = tf32_hi(v[q]);
      float* o = e.out_t + (size_t)(n + q) * e.ldt + m;
      o[0] = hi;
      o[e.plane_t] = v[q] - hi;
    }
  }
}

__global__ void __launch_bounds__(WG_THREADS, 2)
gemm_wgmma_x3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, GemmShape s,
                     GemmEpi e) {
  constexpr int BK = KB_BYTES / 4;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + X3W_OFF_BAR);
  uint64_t* empty = full + X3W_STAGES;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  gemm_entry_guard(e);
  const TileIdx ti = tile_of(s, X3W_BN, BK);

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < X3W_STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      for (int kb = ti.kb0, it = 0; kb < ti.kb1; ++kb, ++it) {
        const int st = it % X3W_STAGES;
        mbar_wait_relaxed(&empty[st], ((it / X3W_STAGES) & 1) ^ 1, 1);
        uint8_t* sA = smem + st * X3W_STAGE;
        mbar_expect_tx(&full[st], X3W_STAGE);
        tma_load_3d(sA, &tmA, &full[st], kb * BK, ti.tm * BM, 0);
        tma_load_3d(sA + X3W_A_BYTES, &tmB, &full[st], kb * BK, ti.tn * X3W_BN, 0);
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;  // rows [64 wg, 64 wg + 64) of the tile
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  reg_fence(acc);
  for (int kb = ti.kb0, it = 0; kb < ti.kb1; ++kb, ++it) {
    const int st = it % X3W_STAGES;
    mbar_wait(&full[st], (it / X3W_STAGES) & 1, 3);
    const uint32_t a_hi = smem_u32(smem + st * X3W_STAGE) + wg * 64 * KB_BYTES;
    const uint32_t a_lo = a_hi + BM * KB_BYTES;
    const uint32_t b_hi = smem_u32(smem + st * X3W_STAGE) + X3W_A_BYTES;
    const uint32_t b_lo = b_hi + X3W_BN * KB_BYTES;
    const uint64_t dah = make_wgmma_desc(a_hi, 0, 1024), dal = make_wgmma_desc(a_lo, 0, 1024);
    const uint64_t dbh = make_wgmma_desc(b_hi, 0, 1024), dbl = make_wgmma_desc(b_lo, 0, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint64_t adv = (uint64_t)((k * 32) >> 4);  // K advances 32 B (8 fp32) per MMA within the swizzled rows
      wgmma_64_tf32(acc, dal + adv, dbh + adv);        // small terms first
      wgmma_64_tf32(acc, dah + adv, dbl + adv);
      wgmma_64_tf32(acc, dah + adv, dbh + adv);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the MMAs of the previous stage have completed: release its slot
    reg_fence(acc);
    if (it > 0) {
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[(it - 1) % X3W_STAGES]);
    }
  }
  wgmma_wait<0>();
  reg_fence(acc);

  // ---- stage the accumulators in the drained operand ring, then the fused epilogue ----
  named_bar(1, 256);
  float* tile = reinterpret_cast<float*>(smem);
  {
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      *reinterpret_cast<float2*>(tile + r0 * X3W_PITCH + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(tile + (r0 + 8) * X3W_PITCH + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  named_bar(1, 256);
  // split-K with counters, as in gemm_x3_kernel: the splits of a tile add in split order
  const bool serial = e.splitk_sem != nullptr && s.splits > 1;
  unsigned* sem = e.splitk_sem + blockIdx.x / s.splits;
  const unsigned split = blockIdx.x % s.splits;
  if (serial) {
    if (threadIdx.x == 0) {
      const long long t0 = clock64();
      while (ld_acquire_u32(sem) != split)
        if (clock64() - t0 > DVT_WATCHDOG_CYCLES) dev_fail(0x5E3u, split);
    }
    named_bar(1, 256);
  }
  epi_tile<true, X3W_BN>(e, s, tile, X3W_PITCH, warp, 8, lane, ti.tm, ti.tn, ti.kb0 < ti.kb_total);
  if (e.out_t) {  // (OUT_F32_SPLIT: never split-K)
    named_bar(1, 256);
    epi_store_t(e, s, tile, X3W_PITCH, ti.tm, ti.tn);
  }
  if (serial) {
    __threadfence();
    named_bar(1, 256);
    if (threadIdx.x == 0) st_release_u32(sem, split + 1 == (unsigned)s.splits ? 0u : split + 1);
  }
}

// ----------------------------------------------------------------------------------------------------
// SIMT debug GEMM (fp32 FMA, 16x16 tiles).  Same epilogue semantics; selected with DVT_GEMM_IMPL=simt or
// dvt_set_debug_impl(1).  It exists so that a broken tensor-core path can be told apart from a broken caller in
// one GPU session; it is never the default.
// ----------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float ld_as_float(const T* p);
template <>
__device__ __forceinline__ float ld_as_float<float>(const float* p) {
  return *p;
}
template <>
__device__ __forceinline__ float ld_as_float<__nv_bfloat16>(const __nv_bfloat16* p) {
  return __bfloat162float(*p);
}

template <typename T>
__global__ void gemm_tn_simt_kernel(const T* __restrict__ A, int lda, const T* __restrict__ B, int ldb, GemmShape s,
                                    GemmEpi e) {
  __shared__ float sa[16][17];
  __shared__ float sb[16][17];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int m = blockIdx.y * 16 + ty;
  const int n = blockIdx.x * 16 + tx;
  float acc = 0.0f;
  for (int k0 = 0; k0 < s.K; k0 += 16) {
    int ka = k0 + tx;
    const T* ap = s.a_mn ? A + (size_t)ka * lda + m : A + (size_t)m * lda + ka;
    sa[ty][tx] = (m < s.M && ka < s.K) ? ld_as_float(ap) + (s.x3 ? ld_as_float(ap + s.plane_a) : 0.0f) : 0.0f;
    int nb = blockIdx.x * 16 + ty;
    const T* bp = s.b_mn ? B + (size_t)ka * ldb + nb : B + (size_t)nb * ldb + ka;
    sb[ty][tx] = (nb < s.N && ka < s.K) ? ld_as_float(bp) + (s.x3 ? ld_as_float(bp + s.plane_b) : 0.0f) : 0.0f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 16; ++k) acc = fmaf(sa[ty][k], sb[tx][k], acc);
    __syncthreads();
  }
  if (m < s.M && n < s.N) {
    if (e.mask_mode == 2) {
      swiglu_bwd_store1(e, m, n, s.N, acc);
    } else {
      const float v = epi_pre(e, m, n, acc);
      epi_post1(e, m, n, v);
      if (e.out_t) {
        const float hi = tf32_hi(v);
        e.out_t[(size_t)n * e.ldt + m] = hi;
        e.out_t[e.plane_t + (size_t)n * e.ldt + m] = v - hi;
      }
    }
  }
}

// SIMT debug form of the RoPE epilogue: one thread per output element computes its own dot product and, on a rotated
// column of a patch row, the one of its partner column n ^ 32 (the other half of the head), then rotates as epi_chunk_rope.
__global__ void gemm_tn_simt_rope_kernel(const __nv_bfloat16* __restrict__ A, int lda, const __nv_bfloat16* __restrict__ B,
                                         int ldb, GemmShape s, GemmEpi e) {
  const int m = blockIdx.y * 16 + threadIdx.y;
  const int n = blockIdx.x * 16 + threadIdx.x;
  if (m >= s.M || n >= s.N) return;
  auto dot = [&](int col) {
    float acc = 0.0f;
    for (int k = 0; k < s.K; ++k)
      acc = fmaf(__bfloat162float(A[(size_t)m * lda + k]), __bfloat162float(B[(size_t)col * ldb + k]), acc);
    return acc + (e.bias ? e.bias[col] : 0.0f);
  };
  float v = dot(n);
  const int t = m % e.rope_ntok;
  if (n < e.rope_cols && t >= e.rope_prefix) {
    const float y = dot(n ^ 32);
    const float* cs = e.rope + (size_t)(t - e.rope_prefix) * 64 + (n & 31);
    v = (n & 32) ? v * cs[0] + y * cs[32] : v * cs[0] - y * cs[32];
  }
  reinterpret_cast<__nv_bfloat16*>(e.out)[(size_t)m * e.ldo + n] = __float2bfloat16_rn(v);
}

template <bool TF32, bool A_MN, bool B_MN, bool GLU = false, bool PLANES = false, bool ROPE = false>
int launch_wgmma(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmShape& s, const GemmEpi& e, cudaStream_t stream) {
  const int tiles = ((s.M + BM - 1) / BM) * ((s.N + WG_BN - 1) / WG_BN) * s.splits;
  if constexpr (ROPE)
    DVT_CUDA_OK(launch_k(s.pdl != 0, gemm_wgmma_rope_kernel, dim3(tiles), dim3(WG_THREADS), (size_t)WG_SMEM, stream, tmA,
                         tmB, s, e));
  else if constexpr (PLANES)
    DVT_CUDA_OK(launch_k(s.pdl != 0, gemm_wgmma_planes_kernel, dim3(tiles), dim3(WG_THREADS), (size_t)WG_SMEM, stream, tmA,
                         tmB, s, e));
  else if constexpr (GLU)
    DVT_CUDA_OK(launch_k(s.pdl != 0, gemm_wgmma_swiglu_bwd_kernel, dim3(tiles), dim3(WG_THREADS), (size_t)WG_SMEM, stream,
                         tmA, tmB, s, e));
  else
    DVT_CUDA_OK(launch_k(s.pdl != 0, gemm_wgmma_kernel<TF32, A_MN, B_MN>, dim3(tiles), dim3(WG_THREADS), (size_t)WG_SMEM,
                         stream, tmA, tmB, s, e));
  count_launch();
  DVT_CUDA_OK(cudaGetLastError());
  return DVT_OK;
}

template <int BN, bool A_MN, bool B_MN>
int launch_x3(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmShape& s, const GemmEpi& e, cudaStream_t stream) {
  const int tiles = ((s.M + BM - 1) / BM) * ((s.N + BN - 1) / BN) * s.splits;
  DVT_CUDA_OK(launch_k(s.pdl != 0, gemm_x3_kernel<BN, A_MN, B_MN>, dim3(tiles), dim3(X3_THREADS),
                       (size_t)X3Smem<BN>::TOTAL, stream, tmA, tmB, s, e));
  count_launch();
  DVT_CUDA_OK(cudaGetLastError());
  return DVT_OK;
}

template <typename K>
int set_smem(K kern, int bytes) {
  DVT_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return DVT_OK;
}

// out[m, n] = sum_k planes[k * plane + m * ldo + n] for k = 0, 1, ... in order (the second step of the ordered split-K)
__global__ void splitk_planes_sum_kernel(const float* __restrict__ planes, int splits, size_t plane, int M, int N, int ldo,
                                         float* __restrict__ out) {
  const int n4 = N >> 2;
  const size_t total = (size_t)M * n4;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int m = (int)(e / n4), n = (int)(e - (size_t)m * n4) * 4;
    const size_t off = (size_t)m * ldo + n;
    float4 acc = __ldg(reinterpret_cast<const float4*>(planes + off));
    for (int k = 1; k < splits; ++k) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(planes + (size_t)k * plane + off));
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    *reinterpret_cast<float4*>(out + off) = acc;
  }
}

}  // namespace

int launch_splitk_planes_sum(const float* planes, int splits, size_t plane, int M, int N, int ldo, float* out,
                             cudaStream_t st) {
  DVT_REQUIRE(planes && out && splits >= 1 && M > 0 && N > 0, "splitk_planes_sum: bad arguments");
  DVT_REQUIRE(N % 4 == 0 && ldo % 4 == 0 && plane % 4 == 0, "splitk_planes_sum: N, ldo and the plane size must be multiples of 4");
  const size_t total = (size_t)M * (N / 4);
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)num_sms() * 8);
  splitk_planes_sum_kernel<<<blocks, 256, 0, st>>>(planes, splits, plane, M, N, ldo, out);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// Opts every instantiation into its dynamic shared memory size.  Called once, outside any stream capture.
int gemm_prepare() {
  static bool done = false;
  if (done) return DVT_OK;
  int rc;
  if ((rc = set_smem(gemm_wgmma_kernel<true, false, false>, WG_SMEM))) return rc;
  if ((rc = set_smem(gemm_wgmma_kernel<false, false, false>, WG_SMEM))) return rc;
  if ((rc = set_smem(gemm_wgmma_kernel<false, false, true>, WG_SMEM))) return rc;
  if ((rc = set_smem(gemm_wgmma_kernel<false, true, true>, WG_SMEM))) return rc;
  if ((rc = set_smem(gemm_wgmma_swiglu_bwd_kernel, WG_SMEM))) return rc;
  if ((rc = set_smem(gemm_wgmma_planes_kernel, WG_SMEM))) return rc;
  if ((rc = set_smem(gemm_wgmma_rope_kernel, WG_SMEM))) return rc;
  if ((rc = set_smem(gemm_wgmma_x3_kernel, X3W_SMEM))) return rc;
  if ((rc = set_smem(gemm_x3_kernel<64, false, true>, X3Smem<64>::TOTAL))) return rc;
  if ((rc = set_smem(gemm_x3_kernel<64, true, true>, X3Smem<64>::TOTAL))) return rc;
  done = true;
  return DVT_OK;
}

int launch_gemm_tn(const void* A, int lda, const void* B, int ldb, TmapDtype dtype, const GemmShape& shape,
                   const GemmEpi& epi_in, cudaStream_t stream) {
  const int impl = debug_impl();
  GemmShape s = shape;
  GemmEpi epi = epi_in;
  if (s.splits < 1) s.splits = 1;
  DVT_REQUIRE(s.M > 0 && s.N > 0 && s.K > 0, "gemm: empty shape M=%d N=%d K=%d", s.M, s.N, s.K);
  DVT_REQUIRE(s.splits == 1 || epi.out_mode == OUT_F32_ATOMIC || epi.out_mode == OUT_F32_PLANES,
              "gemm: split-K needs OUT_F32_ATOMIC or OUT_F32_PLANES");
  const bool planes = epi.out_mode == OUT_F32_PLANES;
  DVT_REQUIRE(!planes || (impl == GEMM_TC && dtype == TMAP_BF16 && s.a_mn && s.b_mn && !s.x3 && epi.out && !epi.bias &&
                          epi.act == ACT_NONE && !epi.mask && !epi.mask_f32 && epi.alpha == 1.0f && !epi.last_col_out &&
                          epi.out_plane >= (size_t)s.M * epi.ldo),
              "gemm: OUT_F32_PLANES needs the tensor-core path, bf16 operands both MN-major, a plain epilogue and planes of at "
              "least M * ldo elements");
  DVT_REQUIRE(epi.out == nullptr || epi.ldo % 4 == 0, "gemm: ldo must be a multiple of 4 (got %d)", epi.ldo);
  DVT_REQUIRE(epi.last_col_out == nullptr || epi.out_mode == OUT_F32_ATOMIC, "gemm: last_col_out needs OUT_F32_ATOMIC");
  epi.last_col_n = epi.last_col_out ? s.N - 1 : -1;
  // the vector post-stage must not straddle the redirected column: keep N-1 in a scalar tail
  DVT_REQUIRE(epi.last_col_out == nullptr || (s.N - 1) % 4 == 0, "gemm: last_col_out needs (N-1) %% 4 == 0 (N=%d)", s.N);
  const bool glu = epi.mask_mode == 2;
  DVT_REQUIRE(!glu || (dtype == TMAP_BF16 && !s.a_mn && s.b_mn && !s.x3 && s.splits == 1 && epi.out_mode == OUT_BF16 &&
                       epi.mask && epi.ldmask % 4 == 0 && epi.ldmask >= 2 * s.N && epi.ldo >= 2 * s.N &&
                       ((reinterpret_cast<uintptr_t>(epi.mask) | reinterpret_cast<uintptr_t>(epi.out)) & 7) == 0),
              "gemm: the SwiGLU-backward epilogue needs bf16 A K-major / B MN-major, no split-K, bf16 output and 8-byte "
              "aligned [M, >= 2N] pre-activation / output with pitches that are multiples of 4");
  // The epilogue reads and writes four consecutive columns at once (float4 / uint2), so every pointer it touches must be
  // aligned for those accesses.  All checks run before any CUDA call: a bad argument is reported, never a fault.
  DVT_REQUIRE(!misaligned(epi.out, epi.out_mode == OUT_BF16 ? 8 : 16),
              "gemm: out must be %d-byte aligned", epi.out_mode == OUT_BF16 ? 8 : 16);
  DVT_REQUIRE(!misaligned(epi.bias, 16) && !misaligned(epi.gamma, 16) && !misaligned(epi.addend, 16),
              "gemm: bias, gamma and addend must be 16-byte aligned");
  DVT_REQUIRE(epi.mask == nullptr || (!misaligned(epi.mask, 8) && epi.ldmask % 4 == 0),
              "gemm: the bf16 mask / GELU pre-activation must be 8-byte aligned with a pitch that is a multiple of 4 (got %d)",
              epi.ldmask);
  DVT_REQUIRE(epi.mask_f32 == nullptr || (!misaligned(epi.mask_f32, 16) && epi.ldmask % 4 == 0),
              "gemm: the fp32 mask must be 16-byte aligned with a pitch that is a multiple of 4 (got %d)", epi.ldmask);
  DVT_REQUIRE(!misaligned(epi.branch, 8), "gemm: branch must be 8-byte aligned");
  DVT_REQUIRE(!misaligned(epi.last_col_out, 4), "gemm: last_col_out must be 4-byte aligned");
  DVT_REQUIRE(epi.out_mode != OUT_F32_SPLIT || epi.out_plane % 4 == 0, "gemm: the lo plane offset must be a multiple of 4");
  DVT_REQUIRE(epi.out_t == nullptr || (epi.out_mode == OUT_F32_SPLIT && s.x3 && !s.a_mn && !s.b_mn && epi.ldt >= s.M),
              "gemm: a transposed output needs OUT_F32_SPLIT of a 3xTF32 product with both operands K-major and ldt >= M");
  const bool rope = epi.rope != nullptr;
  DVT_REQUIRE(!rope || (dtype == TMAP_BF16 && !s.a_mn && !s.b_mn && !s.x3 && s.splits == 1 && epi.out_mode == OUT_BF16 &&
                        epi.act == ACT_NONE && !epi.mask && !epi.mask_f32 && epi.alpha == 1.0f && !epi.last_col_out),
              "gemm: the RoPE epilogue needs bf16 operands both K-major, no split-K and a plain bf16 output");
  DVT_REQUIRE(!rope || (epi.rope_cols > 0 && epi.rope_cols % 64 == 0 && epi.rope_cols <= s.N),
              "gemm: the RoPE columns must be whole 64-wide heads inside N (rope_cols=%d N=%d)", epi.rope_cols, s.N);
  DVT_REQUIRE(!rope || (epi.rope_prefix >= 0 && epi.rope_prefix < epi.rope_ntok),
              "gemm: RoPE needs 0 <= prefix < tokens per image (prefix=%d tokens=%d)", epi.rope_prefix, epi.rope_ntok);
  DVT_REQUIRE(!misaligned(epi.rope, 16), "gemm: the RoPE table must be 16-byte aligned");
  const int elem = dtype == TMAP_BF16 ? 2 : 4;
  DVT_REQUIRE(!misaligned(A, 16) && !misaligned(B, 16), "gemm: operands must be 16-byte aligned");
  if (s.x3) {
    DVT_REQUIRE(dtype == TMAP_F32, "gemm: x3 needs fp32 operands");
    DVT_REQUIRE(!(s.a_mn && !s.b_mn), "gemm: A MN-major with B K-major is not instantiated");
    DVT_REQUIRE((lda * 4) % 16 == 0 && (ldb * 4) % 16 == 0 && (s.plane_a * 4) % 16 == 0 && (s.plane_b * 4) % 16 == 0,
                "gemm: x3 pitches must be multiples of 16 bytes");
  } else {
    DVT_REQUIRE(dtype == TMAP_BF16 || (!s.a_mn && !s.b_mn), "gemm: MN-major operands are implemented for bf16 only");
    DVT_REQUIRE(!(s.a_mn && !s.b_mn), "gemm: A MN-major with B K-major is not instantiated");
    DVT_REQUIRE((lda * elem) % 16 == 0 && (ldb * elem) % 16 == 0,
                "gemm: row pitch must be a multiple of 16 bytes (lda=%d ldb=%d elem=%d)", lda, ldb, elem);
  }

  if (impl == GEMM_SIMT_DEBUG) {
    dim3 grid((s.N + 15) / 16, (s.M + 15) / 16), block(16, 16);
    if (rope)
      gemm_tn_simt_rope_kernel<<<grid, block, 0, stream>>>(reinterpret_cast<const __nv_bfloat16*>(A), lda,
                                                            reinterpret_cast<const __nv_bfloat16*>(B), ldb, s, epi);
    else if (dtype == TMAP_BF16)
      gemm_tn_simt_kernel<__nv_bfloat16><<<grid, block, 0, stream>>>(
          reinterpret_cast<const __nv_bfloat16*>(A), lda, reinterpret_cast<const __nv_bfloat16*>(B), ldb, s, epi);
    else
      gemm_tn_simt_kernel<float><<<grid, block, 0, stream>>>(reinterpret_cast<const float*>(A), lda,
                                                             reinterpret_cast<const float*>(B), ldb, s, epi);
    DVT_CUDA_OK(cudaGetLastError());
    count_launch();
    return DVT_OK;
  }

  {
    int prc = gemm_prepare();
    if (prc) return prc;
  }
  const int bk = KB_BYTES / elem;
  if (s.x3) {
    CUtensorMap tA, tB;
    int rc3;
    // both operands K-major: wgmma (gemm_wgmma_x3_kernel); an MN-major operand: mma.sync (gemm_x3_kernel)
    const bool kk = !s.a_mn && !s.b_mn;
    if (s.a_mn) rc3 = make_tmap_3d(&tA, A, TMAP_F32, (uint64_t)s.M, (uint64_t)s.K, 2, (uint64_t)lda * 4, s.plane_a * 4, 32, 32, 2);
    else rc3 = make_tmap_3d(&tA, A, TMAP_F32, (uint64_t)s.K, (uint64_t)s.M, 2, (uint64_t)lda * 4, s.plane_a * 4, 32, BM, 2);
    if (rc3) return rc3;
    if (s.b_mn) rc3 = make_tmap_3d(&tB, B, TMAP_F32, (uint64_t)s.N, (uint64_t)s.K, 2, (uint64_t)ldb * 4, s.plane_b * 4, 32, 32, 2);
    else rc3 = make_tmap_3d(&tB, B, TMAP_F32, (uint64_t)s.K, (uint64_t)s.N, 2, (uint64_t)ldb * 4, s.plane_b * 4, 32, X3W_BN, 2);
    if (rc3) return rc3;
    if (kk) {
      const int tiles = ((s.M + BM - 1) / BM) * ((s.N + X3W_BN - 1) / X3W_BN) * s.splits;
      DVT_CUDA_OK(launch_k(s.pdl != 0, gemm_wgmma_x3_kernel, dim3(tiles), dim3(WG_THREADS), (size_t)X3W_SMEM, stream, tA, tB,
                           s, epi));
      count_launch();
      DVT_CUDA_OK(cudaGetLastError());
      return DVT_OK;
    }
    if (s.a_mn) return launch_x3<64, true, true>(tA, tB, s, epi, stream);
    return launch_x3<64, false, true>(tA, tB, s, epi, stream);
  }
  CUtensorMap tmA, tmB;
  int rc;
  if (s.a_mn) rc = make_tmap_2d(&tmA, A, dtype, (uint64_t)s.K, (uint64_t)s.M, (uint64_t)lda * elem, bk, 64);
  else rc = make_tmap_2d(&tmA, A, dtype, (uint64_t)s.M, (uint64_t)s.K, (uint64_t)lda * elem, BM, bk);
  if (rc) return rc;
  if (s.b_mn) rc = make_tmap_2d(&tmB, B, dtype, (uint64_t)s.K, (uint64_t)s.N, (uint64_t)ldb * elem, bk, 64);
  else rc = make_tmap_2d(&tmB, B, dtype, (uint64_t)s.N, (uint64_t)s.K, (uint64_t)ldb * elem, WG_BN, bk);
  if (rc) return rc;
  if (dtype == TMAP_F32) return launch_wgmma<true, false, false>(tmA, tmB, s, epi, stream);
  if (glu) return launch_wgmma<false, false, true, true>(tmA, tmB, s, epi, stream);
  if (rope) return launch_wgmma<false, false, false, false, false, true>(tmA, tmB, s, epi, stream);
  if (planes) return launch_wgmma<false, true, true, false, true>(tmA, tmB, s, epi, stream);
  if (s.a_mn) return launch_wgmma<false, true, true>(tmA, tmB, s, epi, stream);
  if (s.b_mn) return launch_wgmma<false, false, true>(tmA, tmB, s, epi, stream);
  return launch_wgmma<false, false, false>(tmA, tmB, s, epi, stream);
}

}  // namespace dvt
