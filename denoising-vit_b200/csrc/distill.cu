// Stage 3 (distillation, reference main_distillation.py): the kernels that training the whole ViT backbone needs on top of
// the stage-2 set (train.cu) -- the LayerScale / residual-branch backward, the backward of the patch embedding and of the
// prefix rows, and the LayerNorm backward of the final norm with its prefix strip.  Every column sum here is a fixed-order
// two-level reduction (per-CTA partials in a caller-provided workspace, then one pass over the partials in CTA order), so
// repeated calls are bit-identical.
#include "common.cuh"
#include "gemm.cuh"

namespace dvt {

// Upper bound on the per-CTA partial rows of the two-level reductions: the workspace holds 2 * kDetChunks rows of C floats.
constexpr int kDetChunks = 128;

static int det_chunks(int rows) { return std::max(1, std::min(kDetChunks, (rows + 63) / 64)); }

// ----------------------------------------------------------------------------------------------------
// LayerScale / residual-branch backward.  Forward: x += gamma * branch, branch = A.B^T + bias.
//   dbranch = gamma * dx (bf16, the dY of the branch GEMMs),  part0[chunk] = sum_rows gamma * dx,
//   part1[chunk] = sum_rows dx * branch.
// Block = 8 row lanes x 32 column lanes, 4 consecutive columns per thread (128 columns per block); blockIdx.y = row chunk.
// gamma == NULL: unit scale (cast + sum only); branch == NULL: no part1; dbranch == NULL: no bf16 output.
// T = bf16: dx is a bf16 matrix (the fixed-order bias gradient of a bf16 dY, dvt_colsum_ordered).
// ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ float4 ld_col4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 ld_col4(const __nv_bfloat16* p) {
  const uint2 v = __ldg(reinterpret_cast<const uint2*>(p));
  const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.x));
  const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.y));
  return make_float4(a.x, a.y, b.x, b.y);
}

template <typename T>
__global__ void __launch_bounds__(256)
branch_bwd_partial_kernel(const T* __restrict__ dx, int ldx, const __nv_bfloat16* __restrict__ branch,
                          const float* __restrict__ gamma, __nv_bfloat16* __restrict__ dbranch, float* __restrict__ part,
                          int rows, int C, int chunks) {
  __shared__ float4 s_b[8][32], s_g[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c = (blockIdx.x * 32 + tx) * 4;
  const int rows_per = (rows + chunks - 1) / chunks;
  const int r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
  float4 ab = make_float4(0.f, 0.f, 0.f, 0.f), ag = ab;
  if (c < C) {
    const float4 g = gamma ? __ldg(reinterpret_cast<const float4*>(gamma + c)) : make_float4(1.f, 1.f, 1.f, 1.f);
    for (int r = r0 + ty; r < r1; r += 8) {
      const float4 d = ld_col4(dx + (size_t)r * ldx + c);
      const float4 gd = make_float4(g.x * d.x, g.y * d.y, g.z * d.z, g.w * d.w);
      ab.x += gd.x; ab.y += gd.y; ab.z += gd.z; ab.w += gd.w;
      if (dbranch) {
        uint2 p;
        p.x = pack_bf16x2(gd.x, gd.y);
        p.y = pack_bf16x2(gd.z, gd.w);
        *reinterpret_cast<uint2*>(dbranch + (size_t)r * C + c) = p;
      }
      if (branch) {
        const uint2 bv = __ldg(reinterpret_cast<const uint2*>(branch + (size_t)r * C + c));
        const float2 b01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&bv.x));
        const float2 b23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&bv.y));
        ag.x = fmaf(d.x, b01.x, ag.x); ag.y = fmaf(d.y, b01.y, ag.y);
        ag.z = fmaf(d.z, b23.x, ag.z); ag.w = fmaf(d.w, b23.y, ag.w);
      }
    }
  }
  s_b[ty][tx] = ab;
  s_g[ty][tx] = ag;
  __syncthreads();
  if (ty == 0 && c < C) {
    float4 sb = s_b[0][tx], sg = s_g[0][tx];
#pragma unroll
    for (int k = 1; k < 8; ++k) {
      const float4 b = s_b[k][tx], q = s_g[k][tx];
      sb.x += b.x; sb.y += b.y; sb.z += b.z; sb.w += b.w;
      sg.x += q.x; sg.y += q.y; sg.z += q.z; sg.w += q.w;
    }
    *reinterpret_cast<float4*>(part + (size_t)blockIdx.y * C + c) = sb;
    if (branch) *reinterpret_cast<float4*>(part + (size_t)(chunks + blockIdx.y) * C + c) = sg;
  }
}

// out0[c] = sum_k part[k, c], out1[c] = sum_k part[chunks + k, c]  (k ascending; out1 optional)
__global__ void partial_final_kernel(const float* __restrict__ part, int chunks, int C, float* __restrict__ out0,
                                     float* __restrict__ out1) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (int k = 0; k < chunks; ++k) s += part[(size_t)k * C + c];
  out0[c] = s;
  if (out1) {
    float t = 0.f;
    for (int k = 0; k < chunks; ++k) t += part[(size_t)(chunks + k) * C + c];
    out1[c] = t;
  }
}

static int launch_partial_final(const float* part, int chunks, int C, float* out0, float* out1, cudaStream_t st) {
  partial_final_kernel<<<(C + 255) / 256, 256, 0, st>>>(part, chunks, C, out0, out1);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

int launch_layerscale_bwd(const float* dx, int ldx, const __nv_bfloat16* branch, const float* gamma, __nv_bfloat16* dbranch,
                          float* dbias, float* dgamma, float* workspace, int rows, int C, cudaStream_t st) {
  DVT_REQUIRE(dx && dbias && workspace && rows > 0 && C > 0, "layerscale_bwd: bad arguments");
  DVT_REQUIRE(C % 4 == 0 && ldx % 4 == 0, "layerscale_bwd: C=%d and ldx=%d must be multiples of 4", C, ldx);
  DVT_REQUIRE(ldx >= C, "layerscale_bwd: row pitch ldx=%d must be >= C=%d", ldx, C);
  DVT_REQUIRE(!misaligned(dx, 16) && !misaligned(gamma, 16) && !misaligned(workspace, 16),
              "layerscale_bwd: dx, gamma and workspace must be 16-byte aligned (float4 accesses)");
  DVT_REQUIRE(!misaligned(branch, 8) && !misaligned(dbranch, 8),
              "layerscale_bwd: branch and dbranch must be 8-byte aligned (4 x bf16 accesses)");
  DVT_REQUIRE(!dgamma || (branch && gamma), "layerscale_bwd: dgamma needs the saved branch and gamma");
  const int chunks = det_chunks(rows);
  branch_bwd_partial_kernel<float><<<dim3((C + 127) / 128, chunks), 256, 0, st>>>(dx, ldx, dgamma ? branch : nullptr, gamma, dbranch,
                                                                          workspace, rows, C, chunks);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return launch_partial_final(workspace, chunks, C, dbias, dgamma, st);
}

// Fixed-order column sums out[c] = sum_rows in[r, c] of a bf16 or fp32 [rows, cols] matrix (the bias gradients of the
// deterministic training step): the partial / final passes of the LayerScale backward without scale or bf16 output.
int launch_colsum_ordered(const void* in, bool bf16, int ld, int rows, int cols, float* out, float* workspace, cudaStream_t st) {
  DVT_REQUIRE(in && out && workspace && rows > 0 && cols > 0, "colsum_ordered: bad arguments");
  DVT_REQUIRE(cols % 4 == 0 && ld % 4 == 0, "colsum_ordered: cols=%d and ld=%d must be multiples of 4", cols, ld);
  DVT_REQUIRE(ld >= cols, "colsum_ordered: row pitch ld=%d must be >= cols=%d", ld, cols);
  DVT_REQUIRE(!misaligned(in, bf16 ? 8 : 16), "colsum_ordered: in must be %d-byte aligned", bf16 ? 8 : 16);
  DVT_REQUIRE(!misaligned(workspace, 16), "colsum_ordered: workspace must be 16-byte aligned");
  const int chunks = det_chunks(rows);
  const dim3 grid((cols + 127) / 128, chunks);
  if (bf16)
    branch_bwd_partial_kernel<__nv_bfloat16><<<grid, 256, 0, st>>>(reinterpret_cast<const __nv_bfloat16*>(in), ld, nullptr,
                                                                  nullptr, nullptr, workspace, rows, cols, chunks);
  else
    branch_bwd_partial_kernel<float><<<grid, 256, 0, st>>>(reinterpret_cast<const float*>(in), ld, nullptr, nullptr, nullptr,
                                                          workspace, rows, cols, chunks);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return launch_partial_final(workspace, chunks, cols, out, nullptr, st);
}

// ----------------------------------------------------------------------------------------------------
// Backward of the patch embedding's token assembly.  Forward (vit.cu): x[b, prefix + p] = patches[b, p] . W^T + bias +
// pos_patch[p]  (OUT_F32_REMAP epilogue), x[b, j < prefix] = prefix_rows[j]  (prefix_rows_kernel).  One thread per
// (token, 4 columns) walks the batch in order:
//   dpatch[b * np + p] = bf16(dx0[b, prefix + p]),  dpos[p] = sum_b dx0[b, prefix + p],  dprefix[j] = sum_b dx0[b, j].
// The bias gradient (sum of dpos over p) follows as a fixed-order column sum.
// ----------------------------------------------------------------------------------------------------
__global__ void embed_bwd_kernel(const float* __restrict__ dx0, int B, int ntok, int prefix, int C,
                                 __nv_bfloat16* __restrict__ dpatch, float* __restrict__ dpos, float* __restrict__ dprefix) {
  const int c4 = C >> 2, np = ntok - prefix;
  const size_t total = (size_t)ntok * c4;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int t = (int)(e / c4), c = (int)(e - (size_t)t * c4) * 4;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int b = 0; b < B; ++b) {
      const float4 d = __ldg(reinterpret_cast<const float4*>(dx0 + ((size_t)b * ntok + t) * C + c));
      acc.x += d.x; acc.y += d.y; acc.z += d.z; acc.w += d.w;
      if (t >= prefix) {
        uint2 p;
        p.x = pack_bf16x2(d.x, d.y);
        p.y = pack_bf16x2(d.z, d.w);
        *reinterpret_cast<uint2*>(dpatch + ((size_t)b * np + (t - prefix)) * C + c) = p;
      }
    }
    float* dst = t < prefix ? dprefix + (size_t)t * C + c : dpos + (size_t)(t - prefix) * C + c;
    *reinterpret_cast<float4*>(dst) = acc;
  }
}

int launch_vit_embed_bwd(const float* dx0, int B, int ntok, int prefix, int C, __nv_bfloat16* dpatch, float* dpos,
                         float* dprefix, float* dbias, float* workspace, cudaStream_t st) {
  DVT_REQUIRE(dx0 && dpatch && dpos && dprefix && dbias && workspace, "vit_embed_bwd: null argument");
  DVT_REQUIRE(B > 0 && prefix >= 1 && ntok > prefix && C > 0 && C % 4 == 0, "vit_embed_bwd: bad shape B=%d ntok=%d prefix=%d C=%d",
              B, ntok, prefix, C);
  DVT_REQUIRE(!misaligned(dx0, 16) && !misaligned(dpos, 16) && !misaligned(dprefix, 16) && !misaligned(workspace, 16),
              "vit_embed_bwd: dx0, dpos, dprefix and workspace must be 16-byte aligned (float4 accesses)");
  DVT_REQUIRE(!misaligned(dpatch, 8), "vit_embed_bwd: dpatch must be 8-byte aligned (4 x bf16 stores)");
  const size_t total = (size_t)ntok * (C / 4);
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)num_sms() * 16);
  embed_bwd_kernel<<<blocks, 256, 0, st>>>(dx0, B, ntok, prefix, C, dpatch, dpos, dprefix);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return launch_layerscale_bwd(dpos, C, nullptr, nullptr, nullptr, dbias, nullptr, workspace, ntok - prefix, C, st);
}

// ----------------------------------------------------------------------------------------------------
// Grouped LayerNorm backward: the mirror of dvt_layernorm's in_group / skip form (final norm + prefix strip).  dy holds the
// compacted rows (o = g * (in_group - skip) + t'), x and dx_accum the full rows (r = g * in_group + skip + t'); prefix rows
// of dx_accum are left as they are.  Same arithmetic as layernorm_bwd_kernel (train.cu); the dgamma / dbeta column sums
// are fixed order: warps add into the CTA's shared partial one after the other, CTAs write their partial rows, and a final
// pass adds them in CTA order.  The grid size depends on the row count only.
// ----------------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_bwd_grouped_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ dy,
                             float* __restrict__ dx_accum, float* __restrict__ part, int out_rows, int C, float eps,
                             int in_group, int skip) {
  extern __shared__ float s_acc[];  // [2 * C]: dgamma | dbeta partials of this CTA
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) s_acc[c] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp_id = threadIdx.x >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int nvec = C >> 2, keep = in_group - skip;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 ag[NV], ab[NV], gm[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    ag[i] = ab[i] = z4;
    gm[i] = lane + 32 * i < nvec ? __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i) : z4;
  }
  for (int o = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; o < out_rows; o += nwarps) {
    const int g = o / keep;
    const size_t row = (size_t)g * in_group + skip + (o - g * keep);
    const float4* xr = reinterpret_cast<const float4*>(x + row * C);
    const float4* dr = reinterpret_cast<const float4*>(dy + (size_t)o * C);
    float4* ar = reinterpret_cast<float4*>(dx_accum + row * C);
    float4 v[NV], d[NV], a[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int idx = lane + 32 * i;
      const bool ok = idx < nvec;
      v[i] = ok ? __ldg(xr + idx) : z4;
      d[i] = ok ? __ldg(dr + idx) : z4;
      a[i] = ok ? ar[idx] : z4;
    }
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    const float mean = warp_sum(sum) / (float)C;
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (lane + 32 * i < nvec) {
        const float p = v[i].x - mean, q = v[i].y - mean, r = v[i].z - mean, s = v[i].w - mean;
        sq += (p * p + q * q) + (r * r + s * s);
      }
    const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      if (lane + 32 * i < nvec) {
        v[i].x = (v[i].x - mean) * rstd; v[i].y = (v[i].y - mean) * rstd;
        v[i].z = (v[i].z - mean) * rstd; v[i].w = (v[i].w - mean) * rstd;
      }
      const float gx = d[i].x * gm[i].x, gy = d[i].y * gm[i].y, gz = d[i].z * gm[i].z, gw = d[i].w * gm[i].w;
      sg += (gx + gy) + (gz + gw);
      sgx += (gx * v[i].x + gy * v[i].y) + (gz * v[i].z + gw * v[i].w);
      ag[i].x = fmaf(d[i].x, v[i].x, ag[i].x); ag[i].y = fmaf(d[i].y, v[i].y, ag[i].y);
      ag[i].z = fmaf(d[i].z, v[i].z, ag[i].z); ag[i].w = fmaf(d[i].w, v[i].w, ag[i].w);
      ab[i].x += d[i].x; ab[i].y += d[i].y; ab[i].z += d[i].z; ab[i].w += d[i].w;
    }
    const float mg = warp_sum(sg) / (float)C, mgx = warp_sum(sgx) / (float)C;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int idx = lane + 32 * i;
      if (idx < nvec) {
        float4 q = a[i];
        q.x += rstd * (d[i].x * gm[i].x - mg - v[i].x * mgx);
        q.y += rstd * (d[i].y * gm[i].y - mg - v[i].y * mgx);
        q.z += rstd * (d[i].z * gm[i].z - mg - v[i].z * mgx);
        q.w += rstd * (d[i].w * gm[i].w - mg - v[i].w * mgx);
        ar[idx] = q;
      }
    }
  }
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {   // warps in order: a fixed summation order inside the CTA
    if (warp_id == w) {
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) {
          float* pg = s_acc + idx * 4;
          float* pb = s_acc + C + idx * 4;
          pg[0] += ag[i].x; pg[1] += ag[i].y; pg[2] += ag[i].z; pg[3] += ag[i].w;
          pb[0] += ab[i].x; pb[1] += ab[i].y; pb[2] += ab[i].z; pb[3] += ab[i].w;
        }
      }
    }
    __syncthreads();
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    part[(size_t)blockIdx.x * C + c] = s_acc[c];
    part[(size_t)(gridDim.x + blockIdx.x) * C + c] = s_acc[C + c];
  }
}

int launch_layernorm_bwd_grouped(const float* x, const float* gamma, const float* dy, float* dx_accum, float* dgamma,
                                 float* dbeta, float* workspace, int rows, int C, float eps, int in_group, int skip,
                                 cudaStream_t st) {
  DVT_REQUIRE(C > 0 && C % 4 == 0 && C <= 2048, "layernorm_bwd_grouped: C=%d unsupported", C);
  DVT_REQUIRE(x && gamma && dy && dx_accum && dgamma && dbeta && workspace, "layernorm_bwd_grouped: null argument");
  DVT_REQUIRE(!misaligned(x, 16) && !misaligned(gamma, 16) && !misaligned(dy, 16) && !misaligned(dx_accum, 16),
              "layernorm_bwd_grouped: x, gamma, dy and dx_accum must be 16-byte aligned (float4 accesses)");
  DVT_REQUIRE(in_group >= 1 && skip >= 0 && skip < in_group && rows % in_group == 0,
              "layernorm_bwd_grouped: bad rows=%d in_group=%d skip=%d", rows, in_group, skip);
  const int out_rows = rows / in_group * (in_group - skip);
  if (out_rows <= 0) return DVT_OK;
  const int nv = (C / 4 + 31) / 32;
  const int blocks = std::min(kDetChunks, (out_rows + 7) / 8);
  const size_t smem = (size_t)2 * C * sizeof(float);
#define DVT_LNG(NV) layernorm_bwd_grouped_kernel<NV><<<blocks, 256, smem, st>>>(x, gamma, dy, dx_accum, workspace, out_rows, C, \
                                                                                eps, in_group, skip)
  if (nv <= 3) DVT_LNG(3);
  else if (nv <= 6) DVT_LNG(6);
  else if (nv <= 8) DVT_LNG(8);
  else if (nv <= 12) DVT_LNG(12);
  else DVT_LNG(16);
#undef DVT_LNG
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return launch_partial_final(workspace, blocks, C, dgamma, dbeta, st);
}

// ----------------------------------------------------------------------------------------------------
// Backward of the 2-D RoPE of the QKV epilogue (gemm.cu epi_chunk_rope), in place on dqkv [M, ld] bf16: on the q and k
// columns of every patch row, with (cos, sin) of the row's patch, per head and d < 32
//   dx[d] = dy[d] cos + dy[d + 32] sin,   dx[d + 32] = dy[d + 32] cos - dy[d] sin      (dx = R^T dy, fp32, one bf16 store)
// One thread per (patch row, head of q or k, 4 frequencies): no reductions, so the result does not depend on the schedule.
// ----------------------------------------------------------------------------------------------------
__global__ void rope_bwd_kernel(__nv_bfloat16* __restrict__ dqkv, int ld, const float* __restrict__ rope, int B, int ntok,
                                int prefix, int qk_heads) {
  const int np = ntok - prefix;
  const int per_row = qk_heads * 8;
  const size_t total = (size_t)B * np * per_row;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(e % per_row);
    const size_t bp = e / per_row;
    const int p = (int)(bp % np), b = (int)(bp / np);
    const int d = (j & 7) * 4;
    __nv_bfloat16* lo = dqkv + ((size_t)b * ntok + prefix + p) * ld + (j >> 3) * 64 + d;
    const uint2 ul = *reinterpret_cast<const uint2*>(lo);
    const uint2 uh = *reinterpret_cast<const uint2*>(lo + 32);
    const float4 c = __ldg(reinterpret_cast<const float4*>(rope + (size_t)p * 64 + d));
    const float4 sn = __ldg(reinterpret_cast<const float4*>(rope + (size_t)p * 64 + 32 + d));
    const float2 l01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ul.x));
    const float2 l23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&ul.y));
    const float2 h01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&uh.x));
    const float2 h23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&uh.y));
    *reinterpret_cast<uint2*>(lo) = make_uint2(pack_bf16x2(l01.x * c.x + h01.x * sn.x, l01.y * c.y + h01.y * sn.y),
                                               pack_bf16x2(l23.x * c.z + h23.x * sn.z, l23.y * c.w + h23.y * sn.w));
    *reinterpret_cast<uint2*>(lo + 32) = make_uint2(pack_bf16x2(h01.x * c.x - l01.x * sn.x, h01.y * c.y - l01.y * sn.y),
                                                    pack_bf16x2(h23.x * c.z - l23.x * sn.z, h23.y * c.w - l23.y * sn.w));
  }
}

int launch_rope_bwd(__nv_bfloat16* dqkv, int ld, const float* rope, int M, int ntok, int prefix, int heads, int head_dim,
                    cudaStream_t st) {
  DVT_REQUIRE(dqkv && rope, "rope_bwd: null argument");
  DVT_REQUIRE(head_dim == 64, "rope_bwd: head_dim must be 64 (got %d)", head_dim);
  DVT_REQUIRE(heads > 0 && M > 0 && ntok > 0 && M % ntok == 0, "rope_bwd: bad shape M=%d tokens=%d heads=%d", M, ntok, heads);
  DVT_REQUIRE(prefix >= 0 && prefix < ntok, "rope_bwd: needs 0 <= prefix < tokens per image (prefix=%d tokens=%d)", prefix,
              ntok);
  DVT_REQUIRE(ld >= 2 * heads * head_dim && ld % 4 == 0, "rope_bwd: ld=%d must be >= 2 * heads * 64 and a multiple of 4", ld);
  DVT_REQUIRE(!misaligned(dqkv, 8) && !misaligned(rope, 16),
              "rope_bwd: dqkv must be 8-byte aligned (4 x bf16 accesses), rope 16-byte aligned (float4 loads)");
  const size_t total = (size_t)(M / ntok) * (ntok - prefix) * (2 * heads) * 8;
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)num_sms() * 16);
  rope_bwd_kernel<<<blocks, 256, 0, st>>>(dqkv, ld, rope, M / ntok, ntok, prefix, 2 * heads);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Token assembly of the training forward: the patch-embed GEMM with the OUT_F32_REMAP epilogue (bias + position) into the
// token rows, then the prefix rows -- the first two steps of vit_forward (vit.cu) on caller-owned tensors.
// ----------------------------------------------------------------------------------------------------
int launch_vit_embed_fwd(const __nv_bfloat16* patches, int Kp, const __nv_bfloat16* w, const float* bias, const float* pos_patch,
                         const float* prefix_rows, int B, int np, int prefix, int C, float* out, cudaStream_t st) {
  // bias may be null (CLIP), pos_patch too (the RoPE ViTs have no absolute position term)
  DVT_REQUIRE(patches && w && prefix_rows && out, "vit_embed_fwd: null argument");
  DVT_REQUIRE(B > 0 && np > 0 && prefix >= 1 && C % 4 == 0 && Kp % 8 == 0, "vit_embed_fwd: bad shape");
  // the GEMM epilogue adds bias and pos_patch and stores out four columns at a time (the GEMM checks them too, by role)
  DVT_REQUIRE(!misaligned(out, 16) && !misaligned(bias, 16) && !misaligned(pos_patch, 16),
              "vit_embed_fwd: out, bias and pos_patch must be 16-byte aligned (float4 accesses)");
  const int ntok = np + prefix;
  GemmEpi e;
  e.bias = bias; e.out_mode = OUT_F32_REMAP; e.out = out; e.ldo = C; e.addend = pos_patch;
  e.rows_per_group = np; e.group_stride = ntok; e.row_offset = prefix;
  GemmShape s{B * np, C, Kp, 1};
  int rc = launch_gemm_tn(patches, Kp, w, Kp, TMAP_BF16, s, e, st);
  if (rc) return rc;
  prefix_rows_kernel<<<B * prefix, 256, 0, st>>>(prefix_rows, out, B, prefix, ntok, C);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

}  // namespace dvt
