// Multi-head self-attention forward for head_dim 64 and 80 on Hopper tensor cores (flash-style, O(N) memory).
//
//   qkv  : bf16 [B, N, 3*C]  (the QKV projection output, C = heads*D; q at col h*D, k at C + h*D, v at 2C + h*D)
//   out  : bf16 [B, N, C]    (col = h*D + d; directly the A operand of the out-projection GEMM)
//   lse  : optional f32 [B, heads, N], log2-domain log-sum-exp of the scaled scores (read by the backward kernel)
//
// One CTA per (query tile of 128 rows, head, image), 9 warps:
//   warps 0-7  two consumer warpgroups, 64 query rows each.  Per key tile of 128 keys: S = Q.K^T (wgmma m64n128k16,
//              Q and K K-major from their TMA tiles), online softmax on the accumulator registers (row max / sum over the
//              four threads that share a row), P -> bf16 registers, O += P.V (wgmma m64n64k16 with A = P from registers,
//              B = V as an MN-major operand straight from its TMA tile).  O stays in registers; its rescaling by
//              exp2(m_old - m_new) is one multiply per element and key tile.
//   warp 8     TMA producer: Q once, then K / V tiles of 128 keys x D through a two-stage ring (3-D tensor map over
//              [3C, N, B]; keys past N are zero-filled and masked out of the softmax).
// head_dim 80: a 160-byte row does not fit one 128-byte swizzle atom.  Every tile is a 64-column slab in the 128-byte
// swizzle (exactly the head_dim-64 tile) followed by a 16-column slab of 32-byte rows in the 32-byte swizzle (a second
// TMA box).  S = Q.K^T takes a fifth k16 step on the tail slabs; O += P.V adds an m64n16k16 wgmma per k16 step whose
// B operand is the V tail slab (MN-major, 32-byte swizzle) and whose 8 accumulators per thread hold O[:, 64:80].
// Reference semantics: timm Attention.forward, restated at evaluation/vitdet/vision_transformer.py:73-91
// (scale d^-0.5, no mask, softmax over keys).
#include "common.cuh"

namespace dvt {

namespace {

constexpr int ATT_BQ = 128;
constexpr int ATT_BK = 128;
constexpr int ATT_THREADS = 288;
constexpr int ATT_MAIN_BYTES = 128 * 128;  // 128 rows x 64 bf16 (128-byte swizzle)

// Shared-memory plan of the head_dim-D kernel: Q, two K stages, two V stages, each [main slab | tail slab].
template <int D>
struct AttCfg {
  static_assert(D == 64 || D == 80, "attention: head_dim 64 or 80");
  static constexpr int TAIL = D - 64;                          // columns in the 32-byte-swizzle slab
  static constexpr int TILE_BYTES = ATT_MAIN_BYTES + 128 * TAIL * 2;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = OFF_Q + TILE_BYTES;             // 2 stages
  static constexpr int OFF_V = OFF_K + 2 * TILE_BYTES;         // 2 stages
  static constexpr int OFF_BAR = OFF_V + 2 * TILE_BYTES;
  static constexpr int SMEM = OFF_BAR + 5 * 8 + 1024;          // + alignment slack
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int D>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap tm_qkv, const __grid_constant__ CUtensorMap tm_tail,
                    __nv_bfloat16* __restrict__ out, int N, int C, float scale_log2e, float* __restrict__ lse) {
  using Cfg = AttCfg<D>;
  constexpr int ATT_TILE_BYTES = Cfg::TILE_BYTES;
  constexpr int ATT_OFF_Q = Cfg::OFF_Q, ATT_OFF_K = Cfg::OFF_K, ATT_OFF_V = Cfg::OFF_V, ATT_OFF_BAR = Cfg::OFF_BAR;
  constexpr int TAIL = Cfg::TAIL;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + ATT_OFF_Q;
  uint8_t* sK = smem + ATT_OFF_K;
  uint8_t* sV = smem + ATT_OFF_V;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ATT_OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;   // [2]
  uint64_t* kv_empty = bars + 3;  // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * ATT_BQ;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int T = (N + ATT_BK - 1) / ATT_BK;  // key tiles

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tm_qkv);
    if constexpr (TAIL > 0) tma_prefetch_desc(&tm_tail);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();     // PDL: the set-up above overlapped the tail of the QKV GEMM
  pdl_trigger();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_expect_tx(q_full, ATT_TILE_BYTES);
      tma_load_3d(sQ, &tm_qkv, q_full, head * D, q0, b);
      if constexpr (TAIL > 0) tma_load_3d(sQ + ATT_MAIN_BYTES, &tm_tail, q_full, head * D + 64, q0, b);
      for (int j = 0; j < T; ++j) {
        const int st = j & 1;
        mbar_wait_relaxed(&kv_empty[st], ((j >> 1) & 1) ^ 1, 10);
        mbar_expect_tx(&kv_full[st], 2 * ATT_TILE_BYTES);
        tma_load_3d(sK + st * ATT_TILE_BYTES, &tm_qkv, &kv_full[st], C + head * D, j * ATT_BK, b);
        tma_load_3d(sV + st * ATT_TILE_BYTES, &tm_qkv, &kv_full[st], 2 * C + head * D, j * ATT_BK, b);
        if constexpr (TAIL > 0) {
          tma_load_3d(sK + st * ATT_TILE_BYTES + ATT_MAIN_BYTES, &tm_tail, &kv_full[st], C + head * D + 64, j * ATT_BK, b);
          tma_load_3d(sV + st * ATT_TILE_BYTES + ATT_MAIN_BYTES, &tm_tail, &kv_full[st], 2 * C + head * D + 64, j * ATT_BK, b);
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  const int t4 = lane & 3;
  // this thread's two query rows (i = 0, 1) within the tile: accumulator rows of the wgmma layout
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint64_t dq = make_wgmma_desc(smem_u32(sQ) + wg * 64 * 128, 0, 1024);
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float ot[TAIL > 0 ? 8 : 1];  // O[:, 64:80] (head_dim 80 only)
#pragma unroll
  for (int i = 0; i < (TAIL > 0 ? 8 : 1); ++i) ot[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY};  // running maximum of s * scale_log2e
  float l_run[2] = {0.f, 0.f};              // this thread's share of the row sums
  mbar_wait(q_full, 0, 14);
  for (int j = 0; j < T; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1, 15);
    // ---- S = Q . K^T ----
    float s[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) s[i] = 0.f;
    const uint64_t dk = make_wgmma_desc(smem_u32(sK + st * ATT_TILE_BYTES), 0, 1024);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_128_bf16<0, 0>(s, dq + (uint64_t)(2 * k), dk + (uint64_t)(2 * k));
    if constexpr (TAIL > 0) {  // fifth k16 step: the 32-byte rows of the tail slabs
      wgmma_128_bf16<0, 0>(s, make_wgmma_desc_sw32(smem_u32(sQ + ATT_MAIN_BYTES) + wg * 64 * 32, 0, 256),
                           make_wgmma_desc_sw32(smem_u32(sK + st * ATT_TILE_BYTES + ATT_MAIN_BYTES), 0, 256));
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    // ---- online softmax (keys >= N: -inf) ----
    const int nval = N - j * ATT_BK;  // valid keys of this tile (>= 1)
    if (nval < ATT_BK) {
#pragma unroll
      for (int jj = 0; jj < 16; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c)
          if (8 * jj + 2 * t4 + c >= nval) s[4 * jj + c] = s[4 * jj + 2 + c] = -INFINITY;
    }
    float alpha[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float mx = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * i], s[4 * jj + 2 * i + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[i], mx * scale_log2e);  // scale > 0: max commutes with the scaling; finite
      alpha[i] = ex2(m_run[i] - m_new);                       // 0 on the first tile (m_run = -inf)
      m_run[i] = m_new;
    }
    uint32_t p[8][4];  // P as the register A operand of P.V: k16 step kk holds keys [16 kk, 16 kk + 16)
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float p0 = ex2(fmaf(s[4 * jj + 2 * i], scale_log2e, -m_run[i]));
        const float p1 = ex2(fmaf(s[4 * jj + 2 * i + 1], scale_log2e, -m_run[i]));
        ls[i] += p0 + p1;
        p[jj >> 1][(jj & 1) * 2 + i] = pack_bf16x2(p0, p1);
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) l_run[i] = l_run[i] * alpha[i] + ls[i];
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
      o[4 * jj] *= alpha[0];
      o[4 * jj + 1] *= alpha[0];
      o[4 * jj + 2] *= alpha[1];
      o[4 * jj + 3] *= alpha[1];
    }
    if constexpr (TAIL > 0) {
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        ot[4 * jj] *= alpha[0];
        ot[4 * jj + 1] *= alpha[0];
        ot[4 * jj + 2] *= alpha[1];
        ot[4 * jj + 3] *= alpha[1];
      }
    }
    // ---- O += P . V  (V rows are keys = the K dimension: 16 keys per MMA = 2048 B) ----
    const uint64_t dv = make_wgmma_desc(smem_u32(sV + st * ATT_TILE_BYTES), 8192, 1024);
    reg_fence(o);
    if constexpr (TAIL > 0) reg_fence(ot);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) wgmma_64_bf16_rs<1>(o, p[kk], dv + (uint64_t)(kk * 2048 >> 4));
    if constexpr (TAIL > 0) {  // V tail slab: 16 keys per MMA = 512 B
      const uint64_t dvt = make_wgmma_desc_sw32(smem_u32(sV + st * ATT_TILE_BYTES + ATT_MAIN_BYTES), 4096, 256);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk) wgmma_16_bf16_rs<1>(ot, p[kk], dvt + (uint64_t)(kk * 512 >> 4));
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
    if constexpr (TAIL > 0) reg_fence(ot);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);  // K / V of this tile are no longer read
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float l = l_run[i];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.0f / l;
    const int q = q0 + row0 + 8 * i;
    if (q < N) {
      // P[q, k] = exp2(s[q, k] * scale_log2e - lse[q]), layout [B, heads, N]
      if (lse && t4 == 0) lse[((size_t)b * gridDim.y + head) * N + q] = m_run[i] + log2f(l);
      __nv_bfloat16* dst = out + ((size_t)b * N + q) * C + head * D + 2 * t4;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(o[4 * jj + 2 * i] * inv, o[4 * jj + 2 * i + 1] * inv);
      if constexpr (TAIL > 0) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj)
          *reinterpret_cast<uint32_t*>(dst + 64 + 8 * jj) =
              pack_bf16x2(ot[4 * jj + 2 * i] * inv, ot[4 * jj + 2 * i + 1] * inv);
      }
    }
  }
}

// ----------------------------------------------------------------------------------------------------
// SIMT debug attention: one warp per (query, head, image); three passes over the keys.  Lane l owns the output
// columns 2l, 2l + 1 and, for head_dim 80, 64 + 2l, 65 + 2l (lanes 0-7).
// ----------------------------------------------------------------------------------------------------
template <int D>
__global__ void attention_simt_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int N,
                                      int C, float scale) {
  constexpr int ATT_D = D;
  constexpr int NPAIR = (D + 63) / 64;  // column pairs per lane
  extern __shared__ float sc[];  // [N] scores
  const int q = blockIdx.x, head = blockIdx.y, b = blockIdx.z;
  const int lane = threadIdx.x;
  const __nv_bfloat16* base = qkv + (size_t)b * N * 3 * C;
  const __nv_bfloat16* qp = base + (size_t)q * 3 * C + head * ATT_D;
  float qv[ATT_D];
#pragma unroll
  for (int d = 0; d < ATT_D; ++d) qv[d] = __bfloat162float(qp[d]);
  float mx = -INFINITY;
  for (int k = lane; k < N; k += 32) {
    const __nv_bfloat16* kp = base + (size_t)k * 3 * C + C + head * ATT_D;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < ATT_D; ++d) s = fmaf(qv[d], __bfloat162float(kp[d]), s);
    s *= scale;
    sc[k] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  float sum = 0.f;
  for (int k = lane; k < N; k += 32) {
    const float p = __expf(sc[k] - mx);
    sc[k] = p;
    sum += p;
  }
  sum = warp_sum(sum);
  __syncwarp();
  float o0[NPAIR], o1[NPAIR];
#pragma unroll
  for (int r = 0; r < NPAIR; ++r) o0[r] = o1[r] = 0.f;
  for (int k = 0; k < N; ++k) {
    const __nv_bfloat16* vp = base + (size_t)k * 3 * C + 2 * C + head * ATT_D;
    const float p = sc[k];
#pragma unroll
    for (int r = 0; r < NPAIR; ++r) {
      const int d = 64 * r + 2 * lane;
      if (d < D) {
        o0[r] = fmaf(p, __bfloat162float(vp[d]), o0[r]);
        o1[r] = fmaf(p, __bfloat162float(vp[d + 1]), o1[r]);
      }
    }
  }
  __nv_bfloat16* dst = out + ((size_t)b * N + q) * C + head * ATT_D;
#pragma unroll
  for (int r = 0; r < NPAIR; ++r) {
    const int d = 64 * r + 2 * lane;
    if (d < D) *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16x2(o0[r] / sum, o1[r] / sum);
  }
}

template <int D>
int launch_attention_d(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int N, int heads, cudaStream_t stream,
                       int impl, float* lse) {
  using Cfg = AttCfg<D>;
  const int C = heads * D;
  // D^-0.5: 0.125 for 64 (exact, the historical literal); rounded to fp32 for 80
  const float scale = D == 64 ? 0.125f : (float)(1.0 / 8.94427190999915878564);
  if (impl == GEMM_SIMT_DEBUG) {
    DVT_REQUIRE(N <= 12000, "attention (simt debug): N=%d too large", N);
    dim3 grid(N, heads, B);
    attention_simt_kernel<D><<<grid, 32, N * sizeof(float), stream>>>(qkv, out, N, C, scale);
    DVT_CUDA_OK(cudaGetLastError());
    count_launch();
    return DVT_OK;
  }
  static bool attr_set = false;  // (attention is never launched inside a stream capture)
  if (!attr_set) {
    DVT_CUDA_OK(cudaFuncSetAttribute(attention_tc_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM));
    attr_set = true;
  }
  CUtensorMap tm, tm_tail;
  int rc = make_tmap_3d(&tm, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, (uint64_t)3 * C * 2,
                        (uint64_t)N * 3 * C * 2, 64, ATT_BK);
  if (rc) return rc;
  if (Cfg::TAIL > 0) {
    rc = make_tmap_3d(&tm_tail, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, (uint64_t)3 * C * 2,
                      (uint64_t)N * 3 * C * 2, Cfg::TAIL, ATT_BK, 1, 32);
    if (rc) return rc;
  } else {
    tm_tail = tm;  // unused
  }
  dim3 grid((N + ATT_BQ - 1) / ATT_BQ, heads, B);
  const float sl2 = scale * 1.4426950408889634f;
  DVT_CUDA_OK(launch_k(false, attention_tc_kernel<D>, grid, dim3(ATT_THREADS), (size_t)Cfg::SMEM, stream, tm, tm_tail,
                       out, N, C, sl2, lse));
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

}  // namespace

// head_dim: 64 or 80 (C = heads * head_dim).  Without lse: the kernel debug_impl() selects.  With lse (training): always
// the tensor-core kernel, the SIMT kernel does not produce the log-sum-exp.
int launch_attention(const __nv_bfloat16* qkv, __nv_bfloat16* out, int B, int N, int heads, cudaStream_t stream,
                     float* lse, int head_dim) {
  DVT_REQUIRE(B > 0 && N > 0 && heads > 0, "attention: bad shape B=%d N=%d heads=%d", B, N, heads);
  DVT_REQUIRE(head_dim == 64 || head_dim == 80, "attention: head_dim %d is not supported (64 or 80)", head_dim);
  const int impl = lse ? GEMM_TC : debug_impl();
  return head_dim == 64 ? launch_attention_d<64>(qkv, out, B, N, heads, stream, impl, lse)
                        : launch_attention_d<80>(qkv, out, B, N, heads, stream, impl, lse);
}

}  // namespace dvt
