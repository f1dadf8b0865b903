// Multi-head self-attention BACKWARD for head_dim 64 and 80 on Hopper tensor cores (flash-style: S and P are recomputed per
// tile from Q, K and the log-sum-exp the forward kernel saved; nothing of size N x N touches HBM).
// Used by the stage-2 training step (reference: loss.backward() through timm Attention inside the `Denoiser` block,
// dvt/models/online_denoiser.py:25-36,90; main_denoiser.py:216-220).
//
//   qkv   : bf16 [B, N, 3C]   forward input (q | k | v, head h at columns h*64)
//   dout  : bf16 [B, N, C]    gradient of the attention output
//   lse   : f32  [B, H, N]    log2-domain log-sum-exp of the scaled scores, written by attention_tc_kernel
//   delta : f32  [B, H, N]    rowsum(dout * out)  (attn_delta_kernel)
//   dqkv  : bf16 [B, N, 3C]   dk, dv written here; dq accumulates in dq_acc f32 [B, N, C] (fp32 reductions)
//
// One CTA per (key tile of 128 keys, head, image), 9 warps; it loops over the query tiles i of 64 queries:
//   warps 0-7  two consumer warpgroups, 64 keys each, all in registers (wgmma accumulator layout, row = key):
//              S^T = K_j Q_i^T and dP^T = V_j dO_i^T (m64n64k16, K-major operands from the TMA tiles);
//              P^T = exp2(S^T * scale*log2e - lse), dS^T = P^T * (dP^T - delta) * scale;
//              dV_j += P^T dO_i and dK_j += dS^T Q_i (A from registers, dO / Q as MN-major B operands);
//              dQ_i += dS K_j over this warpgroup's 64 keys (dS^T staged in swizzled smem as an MN-major A operand,
//              K_j as an MN-major B operand) -> fp32 reductions into dq_acc.
//   warp 8     TMA producer: K_j, V_j once; Q_i and dO_i through a two-stage ring.
// head_dim 80 uses the tile layout of the forward kernel (attention.cu): a 64-column slab in the 128-byte swizzle plus a
// 16-column slab of 32-byte rows in the 32-byte swizzle per tile.  S^T and dP^T take a fifth k16 step on the tail slabs;
// dV, dK and dQ each get an m64n16k16 wgmma per k16 step on the tail slab of dO, Q and K, with 8 more accumulators per
// thread (dK, dV: 40 registers each, still register-resident).
#include "common.cuh"

namespace dvt {

namespace {

constexpr int AB_T = 128;                      // keys per CTA
constexpr int AB_TQ = 64;                      // queries per iteration
constexpr int AB_THREADS = 288;
constexpr int AB_KV_MAIN = 128 * 128;          // bytes of the [128 x 64] bf16 main slab of a K / V tile
constexpr int AB_Q_MAIN = 64 * 128;            // bytes of the [64 x 64] bf16 main slab of a Q / dO tile
constexpr int AB_DS_TILE = 64 * 128;           // one [64 keys x 64 queries] bf16 dS^T tile

template <int D>
struct AbCfg {
  static_assert(D == 64 || D == 80, "attention_bwd: head_dim 64 or 80");
  static constexpr int TAIL = D - 64;          // columns in the 32-byte-swizzle slab
  static constexpr int KV_TILE = AB_KV_MAIN + 128 * TAIL * 2;
  static constexpr int Q_TILE = AB_Q_MAIN + 64 * TAIL * 2;
  static constexpr int OFF_K = 0;
  static constexpr int OFF_V = OFF_K + KV_TILE;
  static constexpr int OFF_Q = OFF_V + KV_TILE;      // 2 stages
  static constexpr int OFF_DO = OFF_Q + 2 * Q_TILE;  // 2 stages
  static constexpr int OFF_DS = OFF_DO + 2 * Q_TILE; // one dS^T tile per warpgroup
  static constexpr int OFF_PT = OFF_DS + 2 * AB_DS_TILE;            // head_dim 80: one P^T tile per warpgroup
  static constexpr int OFF_BAR = OFF_PT + (TAIL > 0 ? 2 * AB_DS_TILE : 0);
  static constexpr int SMEM_TOTAL = OFF_BAR + 5 * 8 + 1024;
};

__device__ __forceinline__ float ab_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// tm_kv_t / tm_q_t / tm_do_t: the 16-column tail boxes (32-byte swizzle) of head_dim 80; unused for 64.
// DQ = false compiles out the dQ part (the dS^T staging that only dQ reads, the dQ wgmma and the fp32 reductions into
// dq_acc): the deterministic backward computes dQ in attention_dq_kernel instead, and dq_acc is not touched.
template <int D, bool DQ = true>
__global__ void __launch_bounds__(AB_THREADS, 1)
attention_bwd_tc_kernel(const __grid_constant__ CUtensorMap tm_kv, const __grid_constant__ CUtensorMap tm_q,
                        const __grid_constant__ CUtensorMap tm_do, const __grid_constant__ CUtensorMap tm_kv_t,
                        const __grid_constant__ CUtensorMap tm_q_t, const __grid_constant__ CUtensorMap tm_do_t,
                        const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                        float* __restrict__ dq_acc, int N, int C, int H, float scale, float scale_log2e) {
  using Cfg = AbCfg<D>;
  constexpr int TAIL = Cfg::TAIL, AB_D = D;
  constexpr int AB_KV_TILE = Cfg::KV_TILE, AB_Q_TILE = Cfg::Q_TILE;
  constexpr int AB_OFF_K = Cfg::OFF_K, AB_OFF_V = Cfg::OFF_V, AB_OFF_Q = Cfg::OFF_Q, AB_OFF_DO = Cfg::OFF_DO;
  constexpr int AB_OFF_DS = Cfg::OFF_DS, AB_OFF_BAR = Cfg::OFF_BAR;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem + AB_OFF_K;
  uint8_t* sV = smem + AB_OFF_V;
  uint8_t* sQ = smem + AB_OFF_Q;
  uint8_t* sDO = smem + AB_OFF_DO;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + AB_OFF_BAR);
  uint64_t* kv_full = bars;
  uint64_t* qd_full = bars + 1;    // [2]
  uint64_t* qd_empty = bars + 3;   // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x;                 // key tile
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int T = (N + AB_TQ - 1) / AB_TQ;    // query tiles

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tm_kv);
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_do);
    if constexpr (TAIL > 0) {
      tma_prefetch_desc(&tm_kv_t);
      tma_prefetch_desc(&tm_q_t);
      tma_prefetch_desc(&tm_do_t);
    }
    mbar_init(kv_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&qd_full[i], 1);
      mbar_init(&qd_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_expect_tx(kv_full, 2 * AB_KV_TILE);
      tma_load_3d(sK, &tm_kv, kv_full, C + head * AB_D, j * AB_T, b);
      tma_load_3d(sV, &tm_kv, kv_full, 2 * C + head * AB_D, j * AB_T, b);
      if constexpr (TAIL > 0) {
        tma_load_3d(sK + AB_KV_MAIN, &tm_kv_t, kv_full, C + head * AB_D + 64, j * AB_T, b);
        tma_load_3d(sV + AB_KV_MAIN, &tm_kv_t, kv_full, 2 * C + head * AB_D + 64, j * AB_T, b);
      }
      for (int i = 0; i < T; ++i) {
        const int st = i & 1;
        mbar_wait_relaxed(&qd_empty[st], ((i >> 1) & 1) ^ 1, 0x60);
        mbar_expect_tx(&qd_full[st], 2 * AB_Q_TILE);
        tma_load_3d(sQ + st * AB_Q_TILE, &tm_q, &qd_full[st], head * AB_D, i * AB_TQ, b);
        tma_load_3d(sDO + st * AB_Q_TILE, &tm_do, &qd_full[st], head * AB_D, i * AB_TQ, b);
        if constexpr (TAIL > 0) {
          tma_load_3d(sQ + st * AB_Q_TILE + AB_Q_MAIN, &tm_q_t, &qd_full[st], head * AB_D + 64, i * AB_TQ, b);
          tma_load_3d(sDO + st * AB_Q_TILE + AB_Q_MAIN, &tm_do_t, &qd_full[st], head * AB_D + 64, i * AB_TQ, b);
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  const int g = lane >> 2, t4 = lane & 3;
  const int krow = (warp & 3) * 16 + g;     // this thread's key rows krow, krow + 8 within the warpgroup's 64 keys
  uint8_t* sDS = smem + AB_OFF_DS + wg * AB_DS_TILE;
  uint8_t* sPT = smem + Cfg::OFF_PT + wg * AB_DS_TILE;  // (head_dim 80 only)
  const size_t stat_base = ((size_t)b * H + head) * N;
  bool key_ok[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) key_ok[i] = j * AB_T + wg * 64 + krow + 8 * i < N;
  const uint64_t dk_a = make_wgmma_desc(smem_u32(sK) + wg * 64 * 128, 0, 1024);     // K rows of this warpgroup, K-major
  const uint64_t dv_a = make_wgmma_desc(smem_u32(sV) + wg * 64 * 128, 0, 1024);
  const uint64_t dk_b = make_wgmma_desc(smem_u32(sK) + wg * 64 * 128, 8192, 1024);  // same rows as an MN-major B (dQ)
  const uint64_t ds_a = make_wgmma_desc(smem_u32(sDS), 8192, 1024);                // dS^T as an MN-major A (dQ)
  float dk[32], dv[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) dk[e] = dv[e] = 0.f;
  constexpr int NT = TAIL > 0 ? 8 : 1;
  float dkt[NT], dvt[NT];  // dK, dV columns 64..79 (head_dim 80 only)
#pragma unroll
  for (int e = 0; e < NT; ++e) dkt[e] = dvt[e] = 0.f;
  mbar_wait(kv_full, 0, 0x63);
  for (int i = 0; i < T; ++i) {
    const int st = i & 1;
    mbar_wait(&qd_full[st], (i >> 1) & 1, 0x61);
    const uint32_t q_addr = smem_u32(sQ + st * AB_Q_TILE), do_addr = smem_u32(sDO + st * AB_Q_TILE);
    uint32_t pa[4][4], da[4][4];  // P^T, dS^T as register A operands (head_dim 64)
    if constexpr (TAIL == 0) {
      float sT[32], dpT[32];
#pragma unroll
      for (int e = 0; e < 32; ++e) sT[e] = dpT[e] = 0.f;
      {
        const uint64_t dq_b = make_wgmma_desc(q_addr, 0, 1024), ddo_b = make_wgmma_desc(do_addr, 0, 1024);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_64_bf16<0, 0>(sT, dk_a + (uint64_t)(2 * k), dq_b + (uint64_t)(2 * k));
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_64_bf16<0, 0>(dpT, dv_a + (uint64_t)(2 * k), ddo_b + (uint64_t)(2 * k));
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(sT);
        reg_fence(dpT);
      }
      // columns of this thread: queries i * 64 + 8 jj + 2 t4 + c; queries past N: lse = +inf makes P (and dS) zero
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float L[2], Dl[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int q = i * AB_TQ + 8 * jj + 2 * t4 + c;
          L[c] = q < N ? __ldg(lse + stat_base + q) : INFINITY;
          Dl[c] = q < N ? __ldg(delta + stat_base + q) : 0.f;
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          float p[2], d[2];
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            p[c] = key_ok[r] ? ab_ex2(fmaf(sT[4 * jj + 2 * r + c], scale_log2e, -L[c])) : 0.f;
            d[c] = p[c] * (dpT[4 * jj + 2 * r + c] - Dl[c]) * scale;
          }
          pa[jj >> 1][(jj & 1) * 2 + r] = pack_bf16x2(p[0], p[1]);
          da[jj >> 1][(jj & 1) * 2 + r] = pack_bf16x2(d[0], d[1]);
        }
      }
      // dS^T -> smem: row = key (128 B = 64 queries, 16-byte chunks swizzled by the row), as the wgmma layouts expect
      if constexpr (DQ) {
        named_bar(1 + wg, 128);  // the previous dQ MMA of this warpgroup has finished reading the buffer
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int row = krow + 8 * r;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
            *reinterpret_cast<uint32_t*>(sDS + row * 128 + ((jj ^ (row & 7)) << 4) + 4 * t4) = da[jj >> 1][(jj & 1) * 2 + r];
        }
      }
    } else {
      // head_dim 80: S^T / dP^T in two halves of 32 queries (m64n32k16: 16 + 16 accumulators instead of 32 + 32), P^T and
      // dS^T written straight to smem; dV / dK then read them from smem as K-major A operands (the same swizzled tiles), so
      // the 16 extra dK / dV accumulators fit in registers.
      named_bar(1 + wg, 128);  // the previous MMAs of this warpgroup have finished reading sDS / sPT
#pragma unroll
      for (int hq = 0; hq < 2; ++hq) {
        float sT[16], dpT[16];
#pragma unroll
        for (int e = 0; e < 16; ++e) sT[e] = dpT[e] = 0.f;
        {
          // 32 query rows further: 4 swizzle atoms (4096 B) in the main slab, 1024 B in the tail slab
          const uint64_t dq_b = make_wgmma_desc(q_addr + hq * 4096, 0, 1024), ddo_b = make_wgmma_desc(do_addr + hq * 4096, 0, 1024);
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_32_bf16<0, 0>(sT, dk_a + (uint64_t)(2 * k), dq_b + (uint64_t)(2 * k));
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_32_bf16<0, 0>(dpT, dv_a + (uint64_t)(2 * k), ddo_b + (uint64_t)(2 * k));
          wgmma_32_bf16<0, 0>(sT, make_wgmma_desc_sw32(smem_u32(sK + AB_KV_MAIN) + wg * 64 * 32, 0, 256),
                              make_wgmma_desc_sw32(q_addr + AB_Q_MAIN + hq * 1024, 0, 256));
          wgmma_32_bf16<0, 0>(dpT, make_wgmma_desc_sw32(smem_u32(sV + AB_KV_MAIN) + wg * 64 * 32, 0, 256),
                              make_wgmma_desc_sw32(do_addr + AB_Q_MAIN + hq * 1024, 0, 256));
          wgmma_commit();
          wgmma_wait<0>();
          reg_fence(sT);
          reg_fence(dpT);
        }
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int ch = 4 * hq + jj;  // 16-byte chunk of the 128-byte row = queries 8 ch .. 8 ch + 7
          float L[2], Dl[2];
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int q = i * AB_TQ + 8 * ch + 2 * t4 + c;
            L[c] = q < N ? __ldg(lse + stat_base + q) : INFINITY;
            Dl[c] = q < N ? __ldg(delta + stat_base + q) : 0.f;
          }
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float p[2], d[2];
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              p[c] = key_ok[r] ? ab_ex2(fmaf(sT[4 * jj + 2 * r + c], scale_log2e, -L[c])) : 0.f;
              d[c] = p[c] * (dpT[4 * jj + 2 * r + c] - Dl[c]) * scale;
            }
            const int row = krow + 8 * r;
            const int off = row * 128 + ((ch ^ (row & 7)) << 4) + 4 * t4;
            *reinterpret_cast<uint32_t*>(sPT + off) = pack_bf16x2(p[0], p[1]);
            *reinterpret_cast<uint32_t*>(sDS + off) = pack_bf16x2(d[0], d[1]);
          }
        }
      }
    }
    if constexpr (DQ || TAIL > 0) {
      fence_async_smem();      // generic-proxy writes of dS^T -> visible to wgmma
      named_bar(1 + wg, 128);
    }
    float dq[DQ ? 32 : 1], dqt[NT];
#pragma unroll
    for (int e = 0; e < (DQ ? 32 : 1); ++e) dq[e] = 0.f;
#pragma unroll
    for (int e = 0; e < NT; ++e) dqt[e] = 0.f;
    {
      const uint64_t q_b = make_wgmma_desc(q_addr, 8192, 1024), do_b = make_wgmma_desc(do_addr, 8192, 1024);
      reg_fence(dv);
      reg_fence(dk);
      wgmma_fence();
      if constexpr (TAIL == 0) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_64_bf16_rs<1>(dv, pa[kk], do_b + (uint64_t)(kk * 128));  // 16 query rows = 2048 B
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_64_bf16_rs<1>(dk, da[kk], q_b + (uint64_t)(kk * 128));
      } else {  // A = P^T / dS^T K-major from smem: +32 B (+2) per k16 step of 16 queries
        const uint64_t pt_a = make_wgmma_desc(smem_u32(sPT), 0, 1024), dst_a = make_wgmma_desc(smem_u32(sDS), 0, 1024);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_64_bf16<0, 1>(dv, pt_a + (uint64_t)(2 * kk), do_b + (uint64_t)(kk * 128));
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_64_bf16<0, 1>(dk, dst_a + (uint64_t)(2 * kk), q_b + (uint64_t)(kk * 128));
      }
      if constexpr (DQ) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_64_bf16<1, 1>(dq, ds_a + (uint64_t)(kk * 128), dk_b + (uint64_t)(kk * 128));  // 16 keys
      }
      if constexpr (TAIL > 0) {  // columns 64..79: MN-major tail slabs, 16 rows = 512 B per k16 step
        reg_fence(dvt);
        reg_fence(dkt);
        const uint64_t dot_b = make_wgmma_desc_sw32(do_addr + AB_Q_MAIN, 4096, 256);
        const uint64_t qt_b = make_wgmma_desc_sw32(q_addr + AB_Q_MAIN, 4096, 256);
        const uint64_t kt_b = make_wgmma_desc_sw32(smem_u32(sK + AB_KV_MAIN) + wg * 64 * 32, 4096, 256);
        const uint64_t pt_a = make_wgmma_desc(smem_u32(sPT), 0, 1024), dst_a = make_wgmma_desc(smem_u32(sDS), 0, 1024);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_16_bf16<0, 1>(dvt, pt_a + (uint64_t)(2 * kk), dot_b + (uint64_t)(kk * 32));
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_16_bf16<0, 1>(dkt, dst_a + (uint64_t)(2 * kk), qt_b + (uint64_t)(kk * 32));
        if constexpr (DQ) {
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_16_bf16<1, 1>(dqt, ds_a + (uint64_t)(kk * 128), kt_b + (uint64_t)(kk * 32));
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(dv);
      reg_fence(dk);
      reg_fence(dq);
      if constexpr (TAIL > 0) {
        reg_fence(dvt);
        reg_fence(dkt);
        reg_fence(dqt);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&qd_empty[st]);  // Q_i / dO_i are no longer read
    // dQ_i partial (this warpgroup's keys): rows = queries 16 (warp & 3) + g + 8 r, columns = d
#pragma unroll
    for (int r = 0; r < 2 && DQ; ++r) {
      const int q = i * AB_TQ + krow + 8 * r;
      if (q < N) {
        float* dst = dq_acc + ((size_t)b * N + q) * C + head * AB_D + 2 * t4;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
          asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + 8 * jj), "f"(dq[4 * jj + 2 * r]),
                       "f"(dq[4 * jj + 2 * r + 1])
                       : "memory");
        if constexpr (TAIL > 0) {
#pragma unroll
          for (int jj = 0; jj < 2; ++jj)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst + 64 + 8 * jj), "f"(dqt[4 * jj + 2 * r]),
                         "f"(dqt[4 * jj + 2 * r + 1])
                         : "memory");
        }
      }
    }
  }
  // dK_j, dV_j (row = key)
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int key = j * AB_T + wg * 64 + krow + 8 * r;
    if (key < N) {
      __nv_bfloat16* dst = dqkv + ((size_t)b * N + key) * 3 * C + head * AB_D + 2 * t4;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        *reinterpret_cast<uint32_t*>(dst + C + 8 * jj) = pack_bf16x2(dk[4 * jj + 2 * r], dk[4 * jj + 2 * r + 1]);
        *reinterpret_cast<uint32_t*>(dst + 2 * C + 8 * jj) = pack_bf16x2(dv[4 * jj + 2 * r], dv[4 * jj + 2 * r + 1]);
      }
      if constexpr (TAIL > 0) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj) {
          *reinterpret_cast<uint32_t*>(dst + C + 64 + 8 * jj) = pack_bf16x2(dkt[4 * jj + 2 * r], dkt[4 * jj + 2 * r + 1]);
          *reinterpret_cast<uint32_t*>(dst + 2 * C + 64 + 8 * jj) = pack_bf16x2(dvt[4 * jj + 2 * r], dvt[4 * jj + 2 * r + 1]);
        }
      }
    }
  }
}

// delta[b, h, q] = sum_d dout[b, q, h*D + d] * out[b, q, h*D + d]; one thread per (b, q, h)
template <int D>
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ dout, const __nv_bfloat16* __restrict__ out,
                                  float* __restrict__ delta, int B, int N, int H) {
  const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (size_t)B * N * H) return;
  const int h = (int)(t % H);
  const size_t bq = t / H;
  const int q = (int)(bq % N), b = (int)(bq / N);
  const uint4* a = reinterpret_cast<const uint4*>(dout + bq * (size_t)H * D + h * D);
  const uint4* o = reinterpret_cast<const uint4*>(out + bq * (size_t)H * D + h * D);
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < D / 8; ++i) {
    const uint4 x = __ldg(a + i), y = __ldg(o + i);
    const __nv_bfloat162* xp = reinterpret_cast<const __nv_bfloat162*>(&x);
    const __nv_bfloat162* yp = reinterpret_cast<const __nv_bfloat162*>(&y);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 xf = __bfloat1622float2(xp[e]), yf = __bfloat1622float2(yp[e]);
      acc = fmaf(xf.x, yf.x, acc);
      acc = fmaf(xf.y, yf.y, acc);
    }
  }
  delta[((size_t)b * H + h) * N + q] = acc;
}

// dqkv[b, q, 0:C] = bf16(dq_acc[b, q, :])
__global__ void attn_dq_cast_kernel(const float* __restrict__ dq_acc, __nv_bfloat16* __restrict__ dqkv, size_t rows, int C) {
  const size_t n4 = rows * (size_t)(C / 4);
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += (size_t)gridDim.x * blockDim.x) {
    const size_t r = e / (C / 4);
    const int c4 = (int)(e - r * (C / 4));
    const float4 v = reinterpret_cast<const float4*>(dq_acc)[e];
    uint2 p;
    p.x = pack_bf16x2(v.x, v.y);
    p.y = pack_bf16x2(v.z, v.w);
    *reinterpret_cast<uint2*>(dqkv + r * 3 * (size_t)C + c4 * 4) = p;
  }
}


// ----------------------------------------------------------------------------------------------------
// Deterministic dQ (the backward under torch.use_deterministic_algorithms): query-major, built like the forward
// attention_tc_kernel.  One CTA per (query tile of 128, head, image), 9 warps:
//   warps 0-7  two consumer warpgroups, 64 queries each.  Q and dO are loaded once; per key tile of 64 keys:
//              S = Q K^T and dP = dO V^T (m64n64k16, K-major operands from the TMA tiles),
//              P = exp2(S * scale*log2e - lse), dS = P * (dP - delta) * scale -> bf16 registers,
//              dQ += dS K (A = dS from registers, B = K as an MN-major operand, as V in the forward's O += P V).
//              dQ stays in registers over all key tiles (fixed order) and is written once, bf16, to dqkv[:, :, 0:C].
//   warp 8     TMA producer: Q, dO once; K / V tiles through a two-stage ring.
// 64-key tiles keep S, dP (32 + 32) and dQ (32, + 8 at head_dim 80) in registers.  head_dim 80: the forward's two-slab
// tiles (128-byte-swizzle main slab + 32-byte-swizzle 16-column tail).  No CTA waits on another.
// ----------------------------------------------------------------------------------------------------
constexpr int DQ_BQ = 128;                     // queries per CTA
constexpr int DQ_BK = 64;                      // keys per tile
constexpr int DQ_Q_MAIN = DQ_BQ * 128;         // bytes of the [128 x 64] main slab of a Q / dO tile
constexpr int DQ_KV_MAIN = DQ_BK * 128;        // bytes of the [64 x 64] main slab of a K / V tile

template <int D>
struct DqCfg {
  static constexpr int TAIL = D - 64;
  static constexpr int Q_TILE = DQ_Q_MAIN + DQ_BQ * TAIL * 2;
  static constexpr int KV_TILE = DQ_KV_MAIN + DQ_BK * TAIL * 2;
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_DO = OFF_Q + Q_TILE;
  static constexpr int OFF_K = OFF_DO + Q_TILE;       // 2 stages
  static constexpr int OFF_V = OFF_K + 2 * KV_TILE;   // 2 stages
  static constexpr int OFF_BAR = OFF_V + 2 * KV_TILE;
  static constexpr int SMEM_TOTAL = OFF_BAR + 5 * 8 + 1024;
  static_assert(Q_TILE % 1024 == 0 && KV_TILE % 1024 == 0, "128-byte-swizzle slabs need 1024-byte alignment");
};

template <int D>
__global__ void __launch_bounds__(AB_THREADS, 1)
attention_dq_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_do,
                    const __grid_constant__ CUtensorMap tm_kv, const __grid_constant__ CUtensorMap tm_q_t,
                    const __grid_constant__ CUtensorMap tm_do_t, const __grid_constant__ CUtensorMap tm_kv_t,
                    const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv, int N,
                    int C, int H, float scale, float scale_log2e) {
  using Cfg = DqCfg<D>;
  constexpr int TAIL = Cfg::TAIL;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + Cfg::OFF_Q;
  uint8_t* sDO = smem + Cfg::OFF_DO;
  uint8_t* sK = smem + Cfg::OFF_K;
  uint8_t* sV = smem + Cfg::OFF_V;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::OFF_BAR);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;   // [2]
  uint64_t* kv_empty = bars + 3;  // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int q0 = blockIdx.x * DQ_BQ;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int T = (N + DQ_BK - 1) / DQ_BK;  // key tiles

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_do);
    tma_prefetch_desc(&tm_kv);
    if constexpr (TAIL > 0) {
      tma_prefetch_desc(&tm_q_t);
      tma_prefetch_desc(&tm_do_t);
      tma_prefetch_desc(&tm_kv_t);
    }
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      mbar_expect_tx(q_full, 2 * Cfg::Q_TILE);
      tma_load_3d(sQ, &tm_q, q_full, head * D, q0, b);
      tma_load_3d(sDO, &tm_do, q_full, head * D, q0, b);
      if constexpr (TAIL > 0) {
        tma_load_3d(sQ + DQ_Q_MAIN, &tm_q_t, q_full, head * D + 64, q0, b);
        tma_load_3d(sDO + DQ_Q_MAIN, &tm_do_t, q_full, head * D + 64, q0, b);
      }
      for (int j = 0; j < T; ++j) {
        const int st = j & 1;
        mbar_wait_relaxed(&kv_empty[st], ((j >> 1) & 1) ^ 1, 0x70);
        mbar_expect_tx(&kv_full[st], 2 * Cfg::KV_TILE);
        uint8_t* k_dst = sK + st * Cfg::KV_TILE;
        uint8_t* v_dst = sV + st * Cfg::KV_TILE;
        tma_load_3d(k_dst, &tm_kv, &kv_full[st], C + head * D, j * DQ_BK, b);
        tma_load_3d(v_dst, &tm_kv, &kv_full[st], 2 * C + head * D, j * DQ_BK, b);
        if constexpr (TAIL > 0) {
          tma_load_3d(k_dst + DQ_KV_MAIN, &tm_kv_t, &kv_full[st], C + head * D + 64, j * DQ_BK, b);
          tma_load_3d(v_dst + DQ_KV_MAIN, &tm_kv_t, &kv_full[st], 2 * C + head * D + 64, j * DQ_BK, b);
        }
      }
    }
    return;
  }

  // ===================== consumer warpgroups =====================
  const int wg = warp >> 2;
  const int t4 = lane & 3;
  const int row0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // this thread's query rows row0, row0 + 8 within the tile
  const size_t stat_base = ((size_t)b * H + head) * N;
  float L[2], Dl[2];  // queries past N: lse = +inf makes P (and dS) zero
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int q = q0 + row0 + 8 * i;
    L[i] = q < N ? __ldg(lse + stat_base + q) : INFINITY;
    Dl[i] = q < N ? __ldg(delta + stat_base + q) : 0.f;
  }
  const uint64_t q_a = make_wgmma_desc(smem_u32(sQ) + wg * 64 * 128, 0, 1024);
  const uint64_t do_a = make_wgmma_desc(smem_u32(sDO) + wg * 64 * 128, 0, 1024);
  constexpr int NT = TAIL > 0 ? 8 : 1;
  float dq[32], dqt[NT];  // dQ columns 0..63 and (head_dim 80) 64..79
#pragma unroll
  for (int e = 0; e < 32; ++e) dq[e] = 0.f;
#pragma unroll
  for (int e = 0; e < NT; ++e) dqt[e] = 0.f;
  mbar_wait(q_full, 0, 0x71);
  for (int j = 0; j < T; ++j) {
    const int st = j & 1;
    mbar_wait(&kv_full[st], (j >> 1) & 1, 0x72);
    const uint32_t k_addr = smem_u32(sK + st * Cfg::KV_TILE), v_addr = smem_u32(sV + st * Cfg::KV_TILE);
    // ---- S = Q K^T, dP = dO V^T ----
    float s[32], dp[32];
#pragma unroll
    for (int e = 0; e < 32; ++e) s[e] = dp[e] = 0.f;
    {
      const uint64_t k_b = make_wgmma_desc(k_addr, 0, 1024), v_b = make_wgmma_desc(v_addr, 0, 1024);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_64_bf16<0, 0>(s, q_a + (uint64_t)(2 * k), k_b + (uint64_t)(2 * k));
      if constexpr (TAIL > 0)  // fifth k16 step: the 32-byte rows of the tail slabs
        wgmma_64_bf16<0, 0>(s, make_wgmma_desc_sw32(smem_u32(sQ + DQ_Q_MAIN) + wg * 64 * 32, 0, 256),
                            make_wgmma_desc_sw32(k_addr + DQ_KV_MAIN, 0, 256));
#pragma unroll
      for (int k = 0; k < 4; ++k) wgmma_64_bf16<0, 0>(dp, do_a + (uint64_t)(2 * k), v_b + (uint64_t)(2 * k));
      if constexpr (TAIL > 0)
        wgmma_64_bf16<0, 0>(dp, make_wgmma_desc_sw32(smem_u32(sDO + DQ_Q_MAIN) + wg * 64 * 32, 0, 256),
                            make_wgmma_desc_sw32(v_addr + DQ_KV_MAIN, 0, 256));
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
      reg_fence(dp);
    }
    // ---- P, dS (keys past N: zero; their K rows are zero-filled too) ----
    const int nval = N - j * DQ_BK;  // valid keys of this tile (>= 1)
    uint32_t ds[4][4];               // dS as the register A operand of dS K: k16 step kk holds keys [16 kk, 16 kk + 16)
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float d[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float p = 8 * jj + 2 * t4 + c < nval ? ab_ex2(fmaf(s[4 * jj + 2 * i + c], scale_log2e, -L[i])) : 0.f;
          d[c] = p * (dp[4 * jj + 2 * i + c] - Dl[i]) * scale;
        }
        ds[jj >> 1][(jj & 1) * 2 + i] = pack_bf16x2(d[0], d[1]);
      }
    }
    // ---- dQ += dS K  (K rows are keys = the K dimension: 16 keys per MMA = 2048 B; tail slab 512 B) ----
    reg_fence(dq);
    if constexpr (TAIL > 0) reg_fence(dqt);
    wgmma_fence();
    {
      const uint64_t k_mn = make_wgmma_desc(k_addr, 8192, 1024);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_64_bf16_rs<1>(dq, ds[kk], k_mn + (uint64_t)(kk * 2048 >> 4));
      if constexpr (TAIL > 0) {
        const uint64_t kt_mn = make_wgmma_desc_sw32(k_addr + DQ_KV_MAIN, 4096, 256);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) wgmma_16_bf16_rs<1>(dqt, ds[kk], kt_mn + (uint64_t)(kk * 512 >> 4));
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dq);
    if constexpr (TAIL > 0) reg_fence(dqt);
    __syncwarp();
    if (lane == 0) mbar_arrive(&kv_empty[st]);  // K / V of this tile are no longer read
  }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int q = q0 + row0 + 8 * i;
    if (q < N) {
      __nv_bfloat16* dst = dqkv + ((size_t)b * N + q) * 3 * C + head * D + 2 * t4;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj)
        *reinterpret_cast<uint32_t*>(dst + 8 * jj) = pack_bf16x2(dq[4 * jj + 2 * i], dq[4 * jj + 2 * i + 1]);
      if constexpr (TAIL > 0) {
#pragma unroll
        for (int jj = 0; jj < 2; ++jj)
          *reinterpret_cast<uint32_t*>(dst + 64 + 8 * jj) = pack_bf16x2(dqt[4 * jj + 2 * i], dqt[4 * jj + 2 * i + 1]);
      }
    }
  }
}

// dq_acc: caller-provided fp32 workspace [B, N, C] (zeroed here); delta: fp32 workspace [B, H, N].
template <int D>
int launch_attention_bwd_d(const __nv_bfloat16* qkv, const __nv_bfloat16* out, const __nv_bfloat16* dout, const float* lse,
                           __nv_bfloat16* dqkv, float* dq_acc, float* delta, int B, int N, int heads, cudaStream_t stream) {
  using Cfg = AbCfg<D>;
  const int C = heads * D;
  static bool attr_set = false;
  if (!attr_set) {
    DVT_CUDA_OK(cudaFuncSetAttribute(attention_bwd_tc_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     Cfg::SMEM_TOTAL));
    attr_set = true;
  }
  DVT_CUDA_OK(cudaMemsetAsync(dq_acc, 0, (size_t)B * N * C * sizeof(float), stream));
  {
    const size_t n = (size_t)B * N * heads;
    attn_delta_kernel<D><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(dout, out, delta, B, N, heads);
    DVT_CUDA_OK(cudaGetLastError());
    count_launch();
  }
  CUtensorMap tkv, tq, td, tkv_t, tq_t, td_t;
  int rc = make_tmap_3d(&tkv, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, (uint64_t)3 * C * 2,
                        (uint64_t)N * 3 * C * 2, 64, AB_T);
  if (rc) return rc;
  rc = make_tmap_3d(&tq, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, (uint64_t)3 * C * 2,
                    (uint64_t)N * 3 * C * 2, 64, AB_TQ);
  if (rc) return rc;
  rc = make_tmap_3d(&td, dout, TMAP_BF16, (uint64_t)C, (uint64_t)N, (uint64_t)B, (uint64_t)C * 2, (uint64_t)N * C * 2, 64,
                    AB_TQ);
  if (rc) return rc;
  if (Cfg::TAIL > 0) {
    rc = make_tmap_3d(&tkv_t, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, (uint64_t)3 * C * 2,
                      (uint64_t)N * 3 * C * 2, Cfg::TAIL, AB_T, 1, 32);
    if (rc) return rc;
    rc = make_tmap_3d(&tq_t, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, (uint64_t)3 * C * 2,
                      (uint64_t)N * 3 * C * 2, Cfg::TAIL, AB_TQ, 1, 32);
    if (rc) return rc;
    rc = make_tmap_3d(&td_t, dout, TMAP_BF16, (uint64_t)C, (uint64_t)N, (uint64_t)B, (uint64_t)C * 2, (uint64_t)N * C * 2,
                      Cfg::TAIL, AB_TQ, 1, 32);
    if (rc) return rc;
  } else {
    tkv_t = tkv; tq_t = tq; td_t = td;  // unused
  }
  // D^-0.5: 0.125 for 64 (exact, the historical literal); rounded to fp32 for 80
  const float scale = D == 64 ? 0.125f : (float)(1.0 / 8.94427190999915878564);
  dim3 grid((N + AB_T - 1) / AB_T, heads, B);
  attention_bwd_tc_kernel<D><<<grid, AB_THREADS, Cfg::SMEM_TOTAL, stream>>>(tkv, tq, td, tkv_t, tq_t, td_t, lse, delta, dqkv,
                                                                             dq_acc, N, C, heads, scale,
                                                                             scale * 1.4426950408889634f);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  attn_dq_cast_kernel<<<num_sms() * 4, 256, 0, stream>>>(dq_acc, dqkv, (size_t)B * N, C);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}


// Deterministic form: delta, then the key-major kernel without its dQ part (dK, dV), then attention_dq_kernel (dQ).
// Every element is written by plain stores from one CTA; no fp32 workspace for dQ.
template <int D>
int launch_attention_bwd_det_d(const __nv_bfloat16* qkv, const __nv_bfloat16* out, const __nv_bfloat16* dout,
                               const float* lse, __nv_bfloat16* dqkv, float* delta, int B, int N, int heads,
                               cudaStream_t stream) {
  using Cfg = AbCfg<D>;
  using DCfg = DqCfg<D>;
  const int C = heads * D;
  static bool attr_set = false;
  if (!attr_set) {
    DVT_CUDA_OK(cudaFuncSetAttribute(attention_bwd_tc_kernel<D, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     Cfg::SMEM_TOTAL));
    DVT_CUDA_OK(cudaFuncSetAttribute(attention_dq_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     DCfg::SMEM_TOTAL));
    attr_set = true;
  }
  {
    const size_t n = (size_t)B * N * heads;
    attn_delta_kernel<D><<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(dout, out, delta, B, N, heads);
    DVT_CUDA_OK(cudaGetLastError());
    count_launch();
  }
  const uint64_t s1q = (uint64_t)3 * C * 2, s2q = (uint64_t)N * 3 * C * 2, s1d = (uint64_t)C * 2, s2d = (uint64_t)N * C * 2;
  // key-major dK / dV kernel: the tensor maps of launch_attention_bwd_d
  CUtensorMap tkv, tq, td, tkv_t, tq_t, td_t;
  int rc = make_tmap_3d(&tkv, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, s1q, s2q, 64, AB_T);
  if (rc) return rc;
  if ((rc = make_tmap_3d(&tq, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, s1q, s2q, 64, AB_TQ))) return rc;
  if ((rc = make_tmap_3d(&td, dout, TMAP_BF16, (uint64_t)C, (uint64_t)N, (uint64_t)B, s1d, s2d, 64, AB_TQ))) return rc;
  // query-major dQ kernel: Q / dO boxes of DQ_BQ rows, K / V boxes of DQ_BK rows
  CUtensorMap gq, gd, gkv, gq_t, gd_t, gkv_t;
  if ((rc = make_tmap_3d(&gq, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, s1q, s2q, 64, DQ_BQ))) return rc;
  if ((rc = make_tmap_3d(&gd, dout, TMAP_BF16, (uint64_t)C, (uint64_t)N, (uint64_t)B, s1d, s2d, 64, DQ_BQ))) return rc;
  if ((rc = make_tmap_3d(&gkv, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, s1q, s2q, 64, DQ_BK))) return rc;
  if (Cfg::TAIL > 0) {
    const int TL = Cfg::TAIL;
    if ((rc = make_tmap_3d(&tkv_t, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, s1q, s2q, TL, AB_T, 1, 32))) return rc;
    if ((rc = make_tmap_3d(&tq_t, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, s1q, s2q, TL, AB_TQ, 1, 32))) return rc;
    if ((rc = make_tmap_3d(&td_t, dout, TMAP_BF16, (uint64_t)C, (uint64_t)N, (uint64_t)B, s1d, s2d, TL, AB_TQ, 1, 32))) return rc;
    if ((rc = make_tmap_3d(&gq_t, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, s1q, s2q, TL, DQ_BQ, 1, 32))) return rc;
    if ((rc = make_tmap_3d(&gd_t, dout, TMAP_BF16, (uint64_t)C, (uint64_t)N, (uint64_t)B, s1d, s2d, TL, DQ_BQ, 1, 32))) return rc;
    if ((rc = make_tmap_3d(&gkv_t, qkv, TMAP_BF16, (uint64_t)3 * C, (uint64_t)N, (uint64_t)B, s1q, s2q, TL, DQ_BK, 1, 32))) return rc;
  } else {
    tkv_t = tkv; tq_t = tq; td_t = td;  // unused
    gq_t = gq; gd_t = gd; gkv_t = gkv;
  }
  const float scale = D == 64 ? 0.125f : (float)(1.0 / 8.94427190999915878564);
  const float sl2 = scale * 1.4426950408889634f;
  attention_bwd_tc_kernel<D, false><<<dim3((N + AB_T - 1) / AB_T, heads, B), AB_THREADS, Cfg::SMEM_TOTAL, stream>>>(
      tkv, tq, td, tkv_t, tq_t, td_t, lse, delta, dqkv, nullptr, N, C, heads, scale, sl2);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  attention_dq_kernel<D><<<dim3((N + DQ_BQ - 1) / DQ_BQ, heads, B), AB_THREADS, DCfg::SMEM_TOTAL, stream>>>(
      gq, gd, gkv, gq_t, gd_t, gkv_t, lse, delta, dqkv, N, C, heads, scale, sl2);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

}  // namespace

// head_dim: 64 or 80 (C = heads * head_dim).
int launch_attention_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* out, const __nv_bfloat16* dout, const float* lse,
                         __nv_bfloat16* dqkv, float* dq_acc, float* delta, int B, int N, int heads, cudaStream_t stream,
                         int head_dim) {
  DVT_REQUIRE(B > 0 && N > 0 && heads > 0, "attention_bwd: bad shape B=%d N=%d heads=%d", B, N, heads);
  DVT_REQUIRE(qkv && out && dout && lse && dqkv && dq_acc && delta, "attention_bwd: null argument");
  DVT_REQUIRE(head_dim == 64 || head_dim == 80, "attention_bwd: head_dim %d is not supported (64 or 80)", head_dim);
  return head_dim == 64 ? launch_attention_bwd_d<64>(qkv, out, dout, lse, dqkv, dq_acc, delta, B, N, heads, stream)
                        : launch_attention_bwd_d<80>(qkv, out, dout, lse, dqkv, dq_acc, delta, B, N, heads, stream);
}

// Deterministic backward (fixed-order dQ): same inputs and dK / dV bits as launch_attention_bwd, no dQ workspace.
int launch_attention_bwd_det(const __nv_bfloat16* qkv, const __nv_bfloat16* out, const __nv_bfloat16* dout, const float* lse,
                             __nv_bfloat16* dqkv, float* delta, int B, int N, int heads, cudaStream_t stream, int head_dim) {
  DVT_REQUIRE(B > 0 && N > 0 && heads > 0, "attention_bwd_det: bad shape B=%d N=%d heads=%d", B, N, heads);
  DVT_REQUIRE(qkv && out && dout && lse && dqkv && delta, "attention_bwd_det: null argument");
  DVT_REQUIRE(head_dim == 64 || head_dim == 80, "attention_bwd_det: head_dim %d is not supported (64 or 80)", head_dim);
  return head_dim == 64 ? launch_attention_bwd_det_d<64>(qkv, out, dout, lse, dqkv, delta, B, N, heads, stream)
                        : launch_attention_bwd_det_d<80>(qkv, out, dout, lse, dqkv, delta, B, N, heads, stream);
}

}  // namespace dvt
