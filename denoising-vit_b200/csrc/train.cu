// Stage 2 (SURVEY.md section 8(f-2)): the bandwidth-bound kernels of the `Denoiser` TRAINING step -- backward of
// LayerNorm, bias gradients, GELU, the distillation loss with its gradient, and AdamW.  The tensor-core parts of the step
// are the bf16 GEMMs of gemm.cu (forward, dgrad with MN-major weights, wgrad with MN-major activations, split-K) and the
// flash-attention forward / backward of attention.cu / attention_bwd.cu.
// Reference: main_denoiser.py:197-221 (forward, MSE + (1 - cosine) loss, loss.backward(), AdamW step) through the timm
// `Block` of dvt/models/online_denoiser.py:25-36 (pre-LN attention + GELU MLP, no LayerScale).
#include "common.cuh"

namespace dvt {

// ----------------------------------------------------------------------------------------------------
// LayerNorm backward.  y = (x - mean) * rstd * gamma + beta  (statistics recomputed from x: cheaper than storing them)
//   dx_accum[r, :] += rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * gamma
//   dgamma += sum_r dy * xhat,  dbeta += sum_r dy
// One warp per row, rows grid-stride over ONE CTA per SM: column partials stay in registers across a warp's rows, are
// combined per CTA in shared memory and leave with one atomic per column and CTA.
// ----------------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(256)
layernorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ dy,
                     float* __restrict__ dx_accum, float* __restrict__ dgamma, float* __restrict__ dbeta, int rows, int C,
                     float eps) {
  extern __shared__ float s_acc[];  // [2 * C]: dgamma | dbeta partials of this CTA
  for (int c = threadIdx.x; c < 2 * C; c += blockDim.x) s_acc[c] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int nvec = C >> 2;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 ag[NV], ab[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) ag[i] = ab[i] = z4;
  float4 gm[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) gm[i] = lane + 32 * i < nvec ? __ldg(reinterpret_cast<const float4*>(gamma) + lane + 32 * i) : z4;
  for (int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += nwarps) {
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * C);
    const float4* dr = reinterpret_cast<const float4*>(dy + (size_t)row * C);
    float4* ar = reinterpret_cast<float4*>(dx_accum + (size_t)row * C);
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
    for (int i = 0; i < NV; ++i) {   // v <- xhat, d stays dy; lanes past the row hold zeros
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
        float4 o = a[i];
        o.x += rstd * (d[i].x * gm[i].x - mg - v[i].x * mgx);
        o.y += rstd * (d[i].y * gm[i].y - mg - v[i].y * mgx);
        o.z += rstd * (d[i].z * gm[i].z - mg - v[i].z * mgx);
        o.w += rstd * (d[i].w * gm[i].w - mg - v[i].w * mgx);
        ar[idx] = o;
      }
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nvec) {
      float* pg = s_acc + idx * 4;
      float* pb = s_acc + C + idx * 4;
      atomicAdd(pg, ag[i].x); atomicAdd(pg + 1, ag[i].y); atomicAdd(pg + 2, ag[i].z); atomicAdd(pg + 3, ag[i].w);
      atomicAdd(pb, ab[i].x); atomicAdd(pb + 1, ab[i].y); atomicAdd(pb + 2, ab[i].z); atomicAdd(pb + 3, ab[i].w);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    atomicAdd(dgamma + c, s_acc[c]);
    atomicAdd(dbeta + c, s_acc[C + c]);
  }
}

int launch_layernorm_bwd(const float* x, const float* gamma, const float* dy, float* dx_accum, float* dgamma, float* dbeta,
                         int rows, int C, float eps, cudaStream_t st) {
  DVT_REQUIRE(C > 0 && C % 4 == 0 && C <= 2048, "layernorm_bwd: C=%d unsupported", C);
  DVT_REQUIRE(x && gamma && dy && dx_accum && dgamma && dbeta, "layernorm_bwd: null argument");
  DVT_REQUIRE(!misaligned(x, 16) && !misaligned(gamma, 16) && !misaligned(dy, 16) && !misaligned(dx_accum, 16),
              "layernorm_bwd: x, gamma, dy and dx_accum must be 16-byte aligned (float4 accesses)");
  if (rows <= 0) return DVT_OK;
  const int nv = (C / 4 + 31) / 32;
  const int blocks = std::min(num_sms(), (rows + 7) / 8);
  const size_t smem = (size_t)2 * C * sizeof(float);
#define DVT_LNB(NV) layernorm_bwd_kernel<NV><<<blocks, 256, smem, st>>>(x, gamma, dy, dx_accum, dgamma, dbeta, rows, C, eps)
  if (nv <= 3) DVT_LNB(3);
  else if (nv <= 6) DVT_LNB(6);
  else if (nv <= 8) DVT_LNB(8);
  else if (nv <= 12) DVT_LNB(12);
  else DVT_LNB(16);
#undef DVT_LNB
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// out[n] += sum_m in[m, n]  (bias gradients).  Block = 32 x 8 threads over a strip of 64 (bf16) / 32 (fp32) columns and
// a chunk of rows; partials meet in shared memory; one atomic per column and block.
// ----------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(256) colsum_kernel(const T* __restrict__ in, int ld, int rows, int cols, float* __restrict__ out) {
  constexpr int W = sizeof(T) == 2 ? 2 : 1;                     // columns per thread
  __shared__ float s_part[8][32 * W];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c0 = (blockIdx.x * 32 + tx) * W;
  const int rows_per = (rows + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per, r1 = min(rows, r0 + rows_per);
  float a0 = 0.f, a1 = 0.f;
  if (c0 < cols) {
    for (int r = r0 + ty; r < r1; r += 8) {
      if constexpr (W == 2) {
        const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(in + (size_t)r * ld + c0);
        a0 += __low2float(v);
        a1 += __high2float(v);
      } else {
        a0 += in[(size_t)r * ld + c0];
      }
    }
  }
  s_part[ty][tx * W] = a0;
  if (W == 2) s_part[ty][tx * W + 1] = a1;
  __syncthreads();
  if (ty == 0 && c0 < cols) {
#pragma unroll
    for (int w = 0; w < W; ++w) {
      float t = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) t += s_part[k][tx * W + w];
      if (c0 + w < cols) atomicAdd(out + c0 + w, t);
    }
  }
}

int launch_colsum(const void* in, bool bf16, int ld, int rows, int cols, float* out, cudaStream_t st) {
  DVT_REQUIRE(in && out && rows > 0 && cols > 0, "colsum: bad arguments");
  DVT_REQUIRE(!bf16 || (cols % 2 == 0 && ld % 2 == 0), "colsum: bf16 input needs even cols / pitch");
  DVT_REQUIRE(ld >= cols, "colsum: row pitch ld=%d must be >= cols=%d", ld, cols);
  DVT_REQUIRE(!misaligned(in, 4), "colsum: in must be 4-byte aligned (bf16x2 / f32 loads)");
  const int strip = bf16 ? 64 : 32;
  const int gx = (cols + strip - 1) / strip;
  const int gy = std::max(1, std::min((rows + 63) / 64, (num_sms() * 4 + gx - 1) / gx));
  if (bf16) colsum_kernel<__nv_bfloat16><<<dim3(gx, gy), 256, 0, st>>>((const __nv_bfloat16*)in, ld, rows, cols, out);
  else colsum_kernel<float><<<dim3(gx, gy), 256, 0, st>>>((const float*)in, ld, rows, cols, out);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// hid = gelu(hpre) (erf GELU, bf16 -> bf16, 8 elements per thread)
__global__ void gelu_bf16_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, size_t n8) {
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n8; e += (size_t)gridDim.x * blockDim.x) {
    const uint4 x = __ldg(in + e);
    const __nv_bfloat162* xp = reinterpret_cast<const __nv_bfloat162*>(&x);
    uint32_t o[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __bfloat1622float2(xp[i]);
      o[i] = pack_bf16x2(gelu_erf(f.x), gelu_erf(f.y));
    }
    out[e] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

int launch_gelu(const __nv_bfloat16* in, __nv_bfloat16* out, size_t n, cudaStream_t st) {
  DVT_REQUIRE(in && out && n % 8 == 0, "gelu: n=%zu must be a multiple of 8", n);
  DVT_REQUIRE(((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 15) == 0, "gelu: 16-byte alignment");
  if (n == 0) return DVT_OK;
  const size_t n8 = n / 8;
  const int blocks = (int)std::min<size_t>((n8 + 255) / 256, (size_t)num_sms() * 16);
  gelu_bf16_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), n8);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Distillation loss of stage 2 (main_denoiser.py:214-217) and its gradient, one warp per row (token):
//   l2 = mean_{rows, C} (pred - tgt)^2,   cos = 1 - mean_rows <pred, tgt> / (max(|pred|, 1e-8) max(|tgt|, 1e-8))
//   dpred = grad_scale * [ 2 (pred - tgt) / (rows C)  -  (tgt / (|p||t|) - cos_r pred / |p|^2) / rows ]
// losses[0..2] += (l2 + cos, l2, cos) contributions (zeroed by the caller).
// ORDERED: CTA k writes its (l2, cos) pair to losses[2 k], losses[2 k + 1] (a workspace) instead; loss_final_kernel adds
// the pairs in CTA order (the fixed-order loss of the deterministic training step).
// ----------------------------------------------------------------------------------------------------
template <int NV, bool ORDERED = false>
__global__ void __launch_bounds__(256)
denoise_loss_kernel(const float* __restrict__ pred, const float* __restrict__ tgt, float* __restrict__ dpred,
                    float* __restrict__ losses, int rows, int C, float grad_scale) {
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int nvec = C >> 2;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  const float inv_nc = 1.f / ((float)rows * (float)C), inv_n = 1.f / (float)rows;
  float acc_l2 = 0.f, acc_cos = 0.f;
  for (int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < rows; row += nwarps) {
    const float4* pr = reinterpret_cast<const float4*>(pred + (size_t)row * C);
    const float4* tr = reinterpret_cast<const float4*>(tgt + (size_t)row * C);
    float4 p[NV], t[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int idx = lane + 32 * i;
      p[i] = idx < nvec ? __ldg(pr + idx) : z4;
      t[i] = idx < nvec ? __ldg(tr + idx) : z4;
    }
    float dot = 0.f, pp = 0.f, tt = 0.f, sse = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      dot += (p[i].x * t[i].x + p[i].y * t[i].y) + (p[i].z * t[i].z + p[i].w * t[i].w);
      pp += (p[i].x * p[i].x + p[i].y * p[i].y) + (p[i].z * p[i].z + p[i].w * p[i].w);
      tt += (t[i].x * t[i].x + t[i].y * t[i].y) + (t[i].z * t[i].z + t[i].w * t[i].w);
      const float a = p[i].x - t[i].x, b = p[i].y - t[i].y, c = p[i].z - t[i].z, d = p[i].w - t[i].w;
      sse += (a * a + b * b) + (c * c + d * d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      dot += __shfl_xor_sync(0xffffffffu, dot, o);
      pp += __shfl_xor_sync(0xffffffffu, pp, o);
      tt += __shfl_xor_sync(0xffffffffu, tt, o);
      sse += __shfl_xor_sync(0xffffffffu, sse, o);
    }
    const float np_ = fmaxf(sqrtf(pp), 1e-8f), nt_ = fmaxf(sqrtf(tt), 1e-8f);  // F.cosine_similarity eps
    const float cosv = dot / (np_ * nt_);
    acc_l2 += sse * inv_nc;
    acc_cos += (1.f - cosv) * inv_n;
    if (dpred) {
      const float k_mse = 2.f * inv_nc * grad_scale;
      const float k_t = -inv_n * grad_scale / (np_ * nt_);
      const float k_p = inv_n * grad_scale * cosv / (np_ * np_);
      float4* dr = reinterpret_cast<float4*>(dpred + (size_t)row * C);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int idx = lane + 32 * i;
        if (idx < nvec) {
          float4 d;
          d.x = k_mse * (p[i].x - t[i].x) + k_t * t[i].x + k_p * p[i].x;
          d.y = k_mse * (p[i].y - t[i].y) + k_t * t[i].y + k_p * p[i].y;
          d.z = k_mse * (p[i].z - t[i].z) + k_t * t[i].z + k_p * p[i].z;
          d.w = k_mse * (p[i].w - t[i].w) + k_t * t[i].w + k_p * p[i].w;
          dr[idx] = d;
        }
      }
    }
  }
  __shared__ float s_part[8][2];
  if (lane == 0) {
    s_part[threadIdx.x >> 5][0] = acc_l2;
    s_part[threadIdx.x >> 5][1] = acc_cos;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float l2 = 0.f, cs = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) {
      l2 += s_part[k][0];
      cs += s_part[k][1];
    }
    if constexpr (ORDERED) {
      losses[2 * blockIdx.x] = l2;
      losses[2 * blockIdx.x + 1] = cs;
    } else {
      atomicAdd(losses + 0, l2 + cs);
      atomicAdd(losses + 1, l2);
      atomicAdd(losses + 2, cs);
    }
  }
}

// losses[1] = sum_k part[2 k], losses[2] = sum_k part[2 k + 1] (k ascending), losses[0] = losses[1] + losses[2]
__global__ void loss_final_kernel(const float* __restrict__ part, int n, float* __restrict__ losses) {
  if (threadIdx.x != 0) return;
  float l2 = 0.f, cs = 0.f;
  for (int k = 0; k < n; ++k) {
    l2 += part[2 * k];
    cs += part[2 * k + 1];
  }
  losses[0] = l2 + cs;
  losses[1] = l2;
  losses[2] = cs;
}

int launch_denoise_loss(const float* pred, const float* tgt, float* dpred, float* losses, int rows, int C, float grad_scale,
                        cudaStream_t st) {
  DVT_REQUIRE(pred && tgt && losses && rows > 0, "denoise_loss: bad arguments");
  DVT_REQUIRE(C > 0 && C % 4 == 0 && C <= 2048, "denoise_loss: C=%d unsupported", C);
  DVT_REQUIRE(!misaligned(pred, 16) && !misaligned(tgt, 16) && !misaligned(dpred, 16),
              "denoise_loss: pred, target and dpred must be 16-byte aligned (float4 accesses)");
  const int nv = (C / 4 + 31) / 32;
  const int blocks = std::min(num_sms() * 4, (rows + 7) / 8);
  DVT_CUDA_OK(cudaMemsetAsync(losses, 0, 3 * sizeof(float), st));
#define DVT_DL(NV) denoise_loss_kernel<NV><<<blocks, 256, 0, st>>>(pred, tgt, dpred, losses, rows, C, grad_scale)
  if (nv <= 3) DVT_DL(3);
  else if (nv <= 6) DVT_DL(6);
  else if (nv <= 8) DVT_DL(8);
  else if (nv <= 12) DVT_DL(12);
  else DVT_DL(16);
#undef DVT_DL
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// Fixed-order form of launch_denoise_loss: the same per-row arithmetic and dpred; workspace f32 [2 * ceil(rows / 8)].
int launch_denoise_loss_ordered(const float* pred, const float* tgt, float* dpred, float* losses, float* workspace, int rows,
                                int C, float grad_scale, cudaStream_t st) {
  DVT_REQUIRE(pred && tgt && losses && workspace && rows > 0, "denoise_loss_ordered: bad arguments");
  DVT_REQUIRE(C > 0 && C % 4 == 0 && C <= 2048, "denoise_loss_ordered: C=%d unsupported", C);
  DVT_REQUIRE(!misaligned(pred, 16) && !misaligned(tgt, 16) && !misaligned(dpred, 16),
              "denoise_loss_ordered: pred, target and dpred must be 16-byte aligned (float4 accesses)");
  const int nv = (C / 4 + 31) / 32;
  const int blocks = std::min(num_sms() * 4, (rows + 7) / 8);
#define DVT_DL(NV) denoise_loss_kernel<NV, true><<<blocks, 256, 0, st>>>(pred, tgt, dpred, workspace, rows, C, grad_scale)
  if (nv <= 3) DVT_DL(3);
  else if (nv <= 6) DVT_DL(6);
  else if (nv <= 8) DVT_DL(8);
  else if (nv <= 12) DVT_DL(12);
  else DVT_DL(16);
#undef DVT_DL
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  loss_final_kernel<<<1, 32, 0, st>>>(workspace, blocks, losses);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Backward of the position-embedding resampling (bicubic, antialias; separable): with the exact fp32 weight matrices
// Wh [h, gh] and Ww [w, gw] of the forward, dgrid[i, j, c] = sum_y sum_x Wh[y, i] Ww[x, j] dout[y, x, c], one axis per
// pass.  One thread per output element sums over its axis in index order: a fixed order, no atomics.
//   dst[o, i, k] = sum_{y < n_out} W[y, i] src[o, y, k]   (src [outer, n_out, inner], dst [outer, n_in, inner])
// ----------------------------------------------------------------------------------------------------
__global__ void resample_axis_bwd_kernel(const float* __restrict__ W, int n_out, int n_in, const float* __restrict__ src,
                                         int outer, int inner, float* __restrict__ dst) {
  const size_t total = (size_t)outer * n_in * inner;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(e % inner);
    const size_t oi = e / inner;
    const int i = (int)(oi % n_in), o = (int)(oi / n_in);
    const float* sp = src + (size_t)o * n_out * inner + k;
    float acc = 0.f;
    for (int y = 0; y < n_out; ++y) acc = fmaf(__ldg(W + (size_t)y * n_in + i), __ldg(sp + (size_t)y * inner), acc);
    dst[e] = acc;
  }
}

static int launch_resample_axis_bwd(const float* W, int n_out, int n_in, const float* src, int outer, int inner, float* dst,
                                    cudaStream_t st) {
  const size_t total = (size_t)outer * n_in * inner;
  const int blocks = (int)std::min<size_t>((total + 255) / 256, (size_t)num_sms() * 16);
  resample_axis_bwd_kernel<<<blocks, 256, 0, st>>>(W, n_out, n_in, src, outer, inner, dst);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

int launch_resample_bwd(const float* wh, const float* ww, const float* dout, float* tmp, float* dgrid, int h, int w, int gh,
                        int gw, int C, cudaStream_t st) {
  DVT_REQUIRE(wh && ww && dout && tmp && dgrid, "resample_bwd: null argument");
  DVT_REQUIRE(h > 0 && w > 0 && gh > 0 && gw > 0 && C > 0, "resample_bwd: bad shape h=%d w=%d gh=%d gw=%d C=%d", h, w, gh, gw, C);
  int rc = launch_resample_axis_bwd(wh, h, gh, dout, 1, w * C, tmp, st);   // tmp [gh, w, C]
  if (rc) return rc;
  return launch_resample_axis_bwd(ww, w, gw, tmp, gh, C, dgrid, st);     // dgrid [gh, gw, C]
}

// ----------------------------------------------------------------------------------------------------
// AdamW over one flat fp32 buffer (torch.optim.AdamW semantics, main_denoiser.py:176-180: decoupled weight decay on
// every parameter, bias-corrected moments, eps outside the square root):
//   p *= 1 - lr wd;  m = b1 m + (1 - b1) g;  v = b2 v + (1 - b2) g^2;  p -= lr / (1 - b1^t) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
// ----------------------------------------------------------------------------------------------------
__global__ void adamw_kernel(float4* __restrict__ p, const float4* __restrict__ g, float4* __restrict__ m,
                             float4* __restrict__ v, size_t n4, float decay, float b1, float b2, float step_size,
                             float inv_bc2_sqrt, float eps) {
  auto upd = [&](float& pp, float gg, float& mm, float& vv) {
    pp *= decay;
    mm = fmaf(b1, mm, (1.f - b1) * gg);
    vv = fmaf(b2, vv, (1.f - b2) * gg * gg);
    pp -= step_size * mm / (sqrtf(vv) * inv_bc2_sqrt + eps);
  };
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n4; e += (size_t)gridDim.x * blockDim.x) {
    float4 pp = p[e], mm = m[e], vv = v[e];
    const float4 gg = g[e];
    upd(pp.x, gg.x, mm.x, vv.x);
    upd(pp.y, gg.y, mm.y, vv.y);
    upd(pp.z, gg.z, mm.z, vv.z);
    upd(pp.w, gg.w, mm.w, vv.w);
    p[e] = pp; m[e] = mm; v[e] = vv;
  }
}

int launch_adamw(float* p, const float* g, float* m, float* v, size_t n, double lr, double beta1, double beta2, double eps,
                 double weight_decay, long long step, cudaStream_t st) {
  DVT_REQUIRE(p && g && m && v, "adamw: null argument");
  DVT_REQUIRE(n % 4 == 0, "adamw: the flat buffer must hold a multiple of 4 elements (got %zu)", n);
  DVT_REQUIRE(step >= 1, "adamw: step counts from 1");
  DVT_REQUIRE(!misaligned(p, 16) && !misaligned(g, 16) && !misaligned(m, 16) && !misaligned(v, 16),
              "adamw: p, g, m and v must be 16-byte aligned (float4 accesses)");
  if (n == 0) return DVT_OK;
  const double bc1 = 1.0 - pow(beta1, (double)step), bc2 = 1.0 - pow(beta2, (double)step);
  const size_t n4 = n / 4;
  const int blocks = (int)std::min<size_t>((n4 + 255) / 256, (size_t)num_sms() * 8);
  adamw_kernel<<<blocks, 256, 0, st>>>((float4*)p, (const float4*)g, (float4*)m, (float4*)v, n4, (float)(1.0 - lr * weight_decay),
                                       (float)beta1, (float)beta2, (float)(lr / bc1), (float)(1.0 / sqrt(bc2)), (float)eps);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

}  // namespace dvt
