// Bandwidth-bound helpers of the frozen-ViT forward (HP-1): LayerNorm (warp per row, float4 loads, shuffle
// reductions), im2col for the patch-embed conv with arbitrary stride, prefix-token rows, SwiGLU gate, casts.
// Reference semantics: timm 1.0.7 VisionTransformer reached from dvt/models/vit_wrapper.py:136-143
// (patch_embed conv with the stride override of vit_wrapper.py:78-79; LayerNorm eps 1e-6; final norm + prefix
// strip + NHWC store replaces the NCHW round trip of main_img_denoising.py:317-323).
#include "common.cuh"

namespace dvt {

// ----------------------------------------------------------------------------------------------------
// LayerNorm: y = (x - mean) / sqrt(var + eps) * gamma + beta, rows of C fp32 (C % 4 == 0, C <= 2048).
// Row mapping: input row r = g * in_group + t (t < in_group).  Rows with t < skip are dropped; output row =
// g * (in_group - skip) + (t - skip).  (skip = number of prefix tokens when writing the patch-only NHWC map.)
// ----------------------------------------------------------------------------------------------------
// NV = float4 per lane (ceil(C / 128)): the row is loaded with NV independent 16-byte loads per lane before any use.
template <typename OutT, int NV>
__global__ void __launch_bounds__(256)
layernorm_kernel(const float* __restrict__ x, int ldx, const float* __restrict__ gamma, const float* __restrict__ beta,
                 OutT* __restrict__ y, int ldy, int rows, int C, float eps, int in_group, int skip) {
  pdl_wait();     // (no-ops unless launched with programmatic stream serialisation)
  pdl_trigger();
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  // grid-stride over rows: the grid is one full wave of CTAs, so there is no partially filled last wave
  for (int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; warp < rows; warp += nwarps) {
  int out_row = warp;
  if (skip > 0) {
    const int g = warp / in_group, t = warp - g * in_group;
    if (t < skip) continue;
    out_row = g * (in_group - skip) + (t - skip);
  }
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)warp * ldx);
  const int nvec = C >> 2;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 v[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = lane + 32 * i;
    v[i] = idx < nvec ? __ldg(xr + idx) : z4;
  }
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  const float mean = warp_sum(sum) / (float)C;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    if (lane + 32 * i < nvec) {
      float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)C + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int idx = lane + 32 * i;
    if (idx < nvec) {
      const float4 g = __ldg(g4 + idx), b = __ldg(b4 + idx);
      float4 o;
      o.x = (v[i].x - mean) * rstd * g.x + b.x;
      o.y = (v[i].y - mean) * rstd * g.y + b.y;
      o.z = (v[i].z - mean) * rstd * g.z + b.z;
      o.w = (v[i].w - mean) * rstd * g.w + b.w;
      if constexpr (sizeof(OutT) == 2) {
        uint2 p;
        p.x = pack_bf16x2(o.x, o.y);
        p.y = pack_bf16x2(o.z, o.w);
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(y) + (size_t)out_row * ldy + idx * 4) = p;
      } else {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(y) + (size_t)out_row * ldy + idx * 4) = o;
      }
    }
  }
  }  // rows
}

// one full wave of CTAs (occupancy x #SM), rows are taken grid-stride
template <typename OutT, int NV>
static void launch_ln_one(int want_blocks, int threads, cudaStream_t stream, const float* x, int ldx, const float* gamma,
                          const float* beta, OutT* y, int ldy, int rows, int C, float eps, int in_group, int skip) {
  static int wave = 0;
  if (wave == 0) {
    int occ = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, layernorm_kernel<OutT, NV>, threads, 0) != cudaSuccess || occ < 1)
      occ = 1;
    wave = occ * num_sms();
  }
  const int blocks = want_blocks < wave ? want_blocks : wave;
  launch_k(false, layernorm_kernel<OutT, NV>, dim3(blocks), dim3(threads), 0, stream, x, ldx, gamma, beta, y, ldy, rows, C,
           eps, in_group, skip);
}

template <typename OutT>
static void launch_ln_nv(int nv, int blocks, int threads, cudaStream_t stream, const float* x, int ldx, const float* gamma,
                         const float* beta, OutT* y, int ldy, int rows, int C, float eps, int in_group, int skip) {
#define DVT_LN(NV) launch_ln_one<OutT, NV>(blocks, threads, stream, x, ldx, gamma, beta, y, ldy, rows, C, eps, in_group, skip)
  if (nv <= 3) DVT_LN(3);
  else if (nv <= 6) DVT_LN(6);
  else if (nv <= 8) DVT_LN(8);
  else if (nv <= 12) DVT_LN(12);
  else DVT_LN(16);
#undef DVT_LN
}

int launch_layernorm(const float* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, bool out_bf16,
                     int rows, int C, float eps, int in_group, int skip, cudaStream_t stream) {
  DVT_REQUIRE(C > 0 && C % 4 == 0 && C <= 2048 && ldx % 4 == 0 && ldy % 4 == 0, "layernorm: C=%d ldx=%d ldy=%d unsupported",
              C, ldx, ldy);
  DVT_REQUIRE(ldx >= C && ldy >= C, "layernorm: row pitches ldx=%d and ldy=%d must be >= C=%d", ldx, ldy, C);
  // skip > 0 compacts whole groups: a partial last group would map its rows past rows / in_group * (in_group - skip)
  DVT_REQUIRE(in_group >= 1 && skip >= 0 && skip < in_group && (skip == 0 || rows % in_group == 0),
              "layernorm: bad in_group=%d / skip=%d for rows=%d (0 <= skip < in_group; rows %% in_group == 0 when skip > 0)",
              in_group, skip, rows);
  // float4 loads of x, gamma and beta; float4 (f32) or uint2 (bf16) stores of y
  DVT_REQUIRE(!misaligned(x, 16), "layernorm: x must be 16-byte aligned");
  DVT_REQUIRE(!misaligned(gamma, 16) && !misaligned(beta, 16), "layernorm: gamma and beta must be 16-byte aligned");
  DVT_REQUIRE(!misaligned(y, out_bf16 ? 8 : 16), "layernorm: y must be %d-byte aligned", out_bf16 ? 8 : 16);
  if (rows <= 0) return DVT_OK;
  const int threads = 256;
  const int blocks = (rows * 32 + threads - 1) / threads;  // upper bound; launch_ln_one caps it at one full wave
  const int nv = (C / 4 + 31) / 32;
  if (out_bf16)
    launch_ln_nv<__nv_bfloat16>(nv, blocks, threads, stream, x, ldx, gamma, beta, (__nv_bfloat16*)y, ldy, rows, C, eps, in_group,
                                skip);
  else
    launch_ln_nv<float>(nv, blocks, threads, stream, x, ldx, gamma, beta, (float*)y, ldy, rows, C, eps, in_group, skip);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// Same row mapping without normalisation (norm=False in get_intermediate_layers): plain strided copy.
__global__ void strip_copy_kernel(const float* __restrict__ x, int ldx, float* __restrict__ y, int ldy, int rows, int C,
                                  int in_group, int skip) {
  const int row = blockIdx.x;
  const int g = row / in_group, t = row - g * in_group;
  if (t < skip) return;
  const int out_row = g * (in_group - skip) + (t - skip);
  for (int c = threadIdx.x; c < C; c += blockDim.x) y[(size_t)out_row * ldy + c] = x[(size_t)row * ldx + c];
}

// ----------------------------------------------------------------------------------------------------
// im2col for Conv2d(3 -> C, kernel P, stride S): x [B, 3, H, W] -> patches bf16 [B*h*w, Kp], column index
// c*P*P + i*P + j (the flattening of the conv weight [C, 3, P, P]); columns >= 3*P*P are zero.
// ----------------------------------------------------------------------------------------------------
// One thread per run of P contiguous source pixels (fixed image, channel, patch and kernel row): index arithmetic once
// per run, 8-byte loads / 4-byte stores when the run is aligned (P, S, W even -- the 14 x 14 patches of the DINOv2 family),
// adjacent threads write adjacent runs of the same patch row.  Run 3 P of every row zero-fills the K padding.
// (Round 1 used one thread per element with 64-bit divisions: 0.204 ms per 32 views, 760 GB/s.)
template <typename InT>
__global__ void im2col_kernel(const InT* __restrict__ x, __nv_bfloat16* __restrict__ out, int B, int H, int W, int P,
                              int S, int h, int w, int Kp, bool vec2) {
  const int runs = 3 * P + 1;
  const size_t total = (size_t)B * h * w * runs;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const size_t row = t / runs;
    const int run = (int)(t - row * runs);
    __nv_bfloat16* o = out + row * Kp;
    if (run == 3 * P) {
      for (int c = 3 * P * P; c < Kp; ++c) o[c] = __float2bfloat16_rn(0.f);
      continue;
    }
    const int c = run / P, i = run - c * P;
    const int pw = (int)(row % w);
    const size_t rq = row / w;
    const int ph = (int)(rq % h);
    const int b = (int)(rq / h);
    const InT* src = x + (((size_t)b * 3 + c) * H + (size_t)ph * S + i) * W + (size_t)pw * S;
    __nv_bfloat16* dst = o + run * P;
    if (vec2) {
      for (int j = 0; j < P; j += 2) {
        __nv_bfloat162 v;
        if constexpr (sizeof(InT) == 2) {
          v = *reinterpret_cast<const __nv_bfloat162*>(src + j);
        } else {
          const float2 f = *reinterpret_cast<const float2*>(src + j);
          v = __floats2bfloat162_rn(f.x, f.y);
        }
        *reinterpret_cast<__nv_bfloat162*>(dst + j) = v;
      }
    } else {
      for (int j = 0; j < P; ++j) {
        float v;
        if constexpr (sizeof(InT) == 2) v = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(src)[j]);
        else v = reinterpret_cast<const float*>(src)[j];
        dst[j] = __float2bfloat16_rn(v);
      }
    }
  }
}

int launch_im2col(const void* x, bool x_bf16, __nv_bfloat16* out, int B, int H, int W, int P, int S, int h, int w,
                  int Kp, cudaStream_t stream) {
  const size_t total = (size_t)B * h * w * (3 * P + 1);
  if (total == (size_t)0 || B == 0) return DVT_OK;
  const int threads = 256;
  const int blocks = (int)((total + threads - 1) / threads < (size_t)num_sms() * 16 ? (total + threads - 1) / threads
                                                                                     : (size_t)num_sms() * 16);
  // paired accesses need even run starts in the source (W, S even) and in the patch matrix (P, Kp even) and aligned bases
  const size_t ea = x_bf16 ? 4 : 8;
  const bool vec2 = P % 2 == 0 && S % 2 == 0 && W % 2 == 0 && Kp % 2 == 0 && (reinterpret_cast<uintptr_t>(x) % ea) == 0 &&
                    (reinterpret_cast<uintptr_t>(out) % 4) == 0;
  if (x_bf16)
    im2col_kernel<__nv_bfloat16><<<blocks, threads, 0, stream>>>((const __nv_bfloat16*)x, out, B, H, W, P, S, h, w, Kp, vec2);
  else
    im2col_kernel<float><<<blocks, threads, 0, stream>>>((const float*)x, out, B, H, W, P, S, h, w, Kp, vec2);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// prefix rows (cls [+pos] and register tokens), precomputed as [prefix, C]; broadcast to every image of the batch
__global__ void prefix_rows_kernel(const float* __restrict__ prefix_rows, float* __restrict__ x, int B, int prefix,
                                   int ntok, int C) {
  const int b = blockIdx.x / prefix, p = blockIdx.x % prefix;
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    x[((size_t)b * ntok + p) * C + c] = prefix_rows[(size_t)p * C + c];
}

// SwiGLU (timm SwiGLUPacked, gate_last=False): out[m, j] = silu(h[m, j]) * h[m, j + Hh], h bf16 [M, 2*Hh]
__global__ void swiglu_kernel(const __nv_bfloat16* __restrict__ hin, __nv_bfloat16* __restrict__ out, size_t M, int Hh) {
  const size_t total = M * Hh;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t m = e / Hh;
    const int j = (int)(e - m * Hh);
    const float a = __bfloat162float(hin[m * 2 * Hh + j]);
    const float b = __bfloat162float(hin[m * 2 * Hh + Hh + j]);
    out[e] = __float2bfloat16_rn(a / (1.f + __expf(-a)) * b);
  }
}

// swiglu_kernel on caller-owned tensors (the training forward): the same launch as the inference forward in vit.cu, so both
// produce the same bits
int launch_swiglu(const __nv_bfloat16* hin, __nv_bfloat16* out, size_t M, int Hh, cudaStream_t st) {
  DVT_REQUIRE(hin && out && Hh > 0, "swiglu: bad arguments");
  if (M == 0) return DVT_OK;
  swiglu_kernel<<<num_sms() * 8, 256, 0, st>>>(hin, out, M, Hh);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ in, __nv_bfloat16* __restrict__ out, size_t n) {
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x)
    out[e] = __float2bfloat16_rn(in[e]);
}

// conv weight [C, 3*P*P] fp32 -> bf16 [C, Kp] zero padded
__global__ void pad_cast_rows_kernel(const float* __restrict__ in, int K, __nv_bfloat16* __restrict__ out, int Kp,
                                     size_t rows) {
  const size_t total = rows * Kp;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t r = e / Kp;
    const int c = (int)(e - r * Kp);
    out[e] = __float2bfloat16_rn(c < K ? in[r * K + c] : 0.f);
  }
}

}  // namespace dvt
