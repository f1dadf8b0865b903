// Dense-task linear probe (NYU depth): the full-resolution parts of the BNHead bin-classification head (classify=True,
// UD bins, linear norm), of the loss resize and of whole-image evaluation with flip test-time augmentation.
//
// Every resize is ATen's upsample_bilinear2d with align_corners=False in fp32 (the SegTap / seg_lerp arithmetic of
// seg.cu).  The head relies on two identities: the 1x1 conv is linear and the bilinear weights of a pixel sum to 1, so
// conv(upsample(x)) = upsample(conv(x)); the caller computes the n_bins logits at the low resolution and these kernels
// interpolate them per pixel.  No float atomics: every sum has a fixed order, so repeated calls are bit-identical.
#include "common.cuh"

#include <algorithm>

namespace dvt {

namespace {

constexpr int kDepthWarps = 8;
constexpr int kDepthTile = 2;   // low-resolution cells per CTA along each axis (head backward)
constexpr int kDepthNb = kDepthTile + 2;
constexpr int kDepthEvalBlocks = 128;  // per image; fixed, so the partial sums do not depend on the device
constexpr int kDepthEvalThreads = 256;
constexpr int kDepthSums = 10;

// Per pixel: r_k = bilinear(logits)_k, a_k = relu(r_k) + 0.1 (0 for the padding lanes k >= K), S = sum_k a_k,
// depth = sum_k (a_k / S) bin_k (the reference's normalise-then-einsum order).  Returns depth, writes r, a and S.
template <int KV>
__device__ __forceinline__ float depth_pixel(const SegTap& ty, const SegTap& tx, const float* c00, const float* c01,
                                             const float* c10, const float* c11, const float* binv, int K, int lane,
                                             float* r, float* a, float& S) {
  float s = 0.f;
#pragma unroll
  for (int v = 0; v < KV; ++v) {
    const int k = lane + 32 * v;
    r[v] = k < K ? seg_lerp(ty, tx, c00[k], c01[k], c10[k], c11[k]) : 0.f;
    a[v] = k < K ? fmaxf(r[v], 0.f) + 0.1f : 0.f;
    s += a[v];
  }
  S = warp_sum_f(s);
  float d = 0.f;
#pragma unroll
  for (int v = 0; v < KV; ++v) d += (a[v] / S) * binv[v];
  return warp_sum_f(d);
}

}  // namespace

// ----------------------------------------------------------------------------------------------------
// Head forward: one warp per pixel of the up x resolution map, lanes over the bins (k = lane + 32 v).
// ----------------------------------------------------------------------------------------------------
template <int KV>
__global__ void __launch_bounds__(kDepthWarps * 32) depth_head_fwd_kernel(const float* __restrict__ logits, int B, int h,
                                                                          int w, int K, int up, const float* __restrict__ bins,
                                                                          float* __restrict__ depth) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Hu = h * up, Wu = w * up;
  const float sy = (float)h / (float)Hu, sx = (float)w / (float)Wu;
  float binv[KV];
#pragma unroll
  for (int v = 0; v < KV; ++v) binv[v] = lane + 32 * v < K ? __ldg(bins + lane + 32 * v) : 0.f;
  const long long n = (long long)B * Hu * Wu;
  for (long long e = (long long)blockIdx.x * kDepthWarps + warp; e < n; e += (long long)gridDim.x * kDepthWarps) {
    const int b = (int)(e / ((long long)Hu * Wu));
    const int p = (int)(e % ((long long)Hu * Wu));
    const int y = p / Wu, x = p % Wu;
    const SegTap ty = seg_tap(y, h, sy), tx = seg_tap(x, w, sx);
    const float* img = logits + (size_t)b * h * w * K;
    float r[KV], a[KV], S;
    const float d = depth_pixel<KV>(ty, tx, img + ((size_t)ty.i0 * w + tx.i0) * K, img + ((size_t)ty.i0 * w + tx.i1) * K,
                                    img + ((size_t)ty.i1 * w + tx.i0) * K, img + ((size_t)ty.i1 * w + tx.i1) * K, binv, K,
                                    lane, r, a, S);
    if (lane == 0) depth[e] = d;
  }
}

// ----------------------------------------------------------------------------------------------------
// Head backward, gathered at the low resolution: CTA = (2 x 2 cells, image), as seg_upsample_ce_kernel.  It walks every
// pixel whose 4-tap footprint touches one of its cells (one warp per pixel), recomputes the pixel's logits from the 4 x 4
// neighbourhood of cells staged in shared memory, and adds w_tap * d r_k, with d r_k = g (bin_k - depth) / S for r_k > 0
// (relu'(0) = 0), into per-warp register accumulators; the warps' accumulators are added in warp order.
// ----------------------------------------------------------------------------------------------------
template <int KV>
__global__ void __launch_bounds__(kDepthWarps * 32) depth_head_bwd_kernel(const float* __restrict__ logits, int h, int w, int K,
                                                                          int up, const float* __restrict__ bins,
                                                                          const float* __restrict__ ddepth,
                                                                          float* __restrict__ dlogits) {
  extern __shared__ float depth_sm[];  // [nb cells][K] neighbourhood, later [warps][tile cells][K] partial sums
  __shared__ int s_lo[2], s_hi[2];
  const int b = blockIdx.z, i0 = blockIdx.y * kDepthTile, j0 = blockIdx.x * kDepthTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Hu = h * up, Wu = w * up;
  const float sy = (float)h / (float)Hu, sx = (float)w / (float)Wu;
  if (threadIdx.x < 2) {
    s_lo[threadIdx.x] = 1 << 30;
    s_hi[threadIdx.x] = -1;
  }
  const float* src = logits + (size_t)b * h * w * K;
  for (int e = threadIdx.x; e < kDepthNb * kDepthNb * K; e += blockDim.x) {
    const int k = e % K, c = e / K;
    const int r = i0 - 1 + c / kDepthNb, q = j0 - 1 + c % kDepthNb;
    if (r >= 0 && r < h && q >= 0 && q < w) depth_sm[e] = __ldg(src + ((size_t)r * w + q) * K + k);
  }
  __syncthreads();
  for (int y = threadIdx.x; y < Hu; y += blockDim.x) {
    const int r = seg_tap(y, h, sy).i0;
    if (r >= i0 - 1 && r <= i0 + kDepthTile - 1) {
      atomicMin(&s_lo[0], y);
      atomicMax(&s_hi[0], y);
    }
  }
  for (int x = threadIdx.x; x < Wu; x += blockDim.x) {
    const int q = seg_tap(x, w, sx).i0;
    if (q >= j0 - 1 && q <= j0 + kDepthTile - 1) {
      atomicMin(&s_lo[1], x);
      atomicMax(&s_hi[1], x);
    }
  }
  __syncthreads();
  const int ylo = s_lo[0], xlo = s_lo[1];
  const int ny = s_hi[0] - ylo + 1, nx = s_hi[1] - xlo + 1;
  const int npix = (ny > 0 && nx > 0) ? ny * nx : 0;

  float binv[KV];
#pragma unroll
  for (int v = 0; v < KV; ++v) binv[v] = lane + 32 * v < K ? __ldg(bins + lane + 32 * v) : 0.f;
  float acc[kDepthTile][kDepthTile][KV];
#pragma unroll
  for (int a = 0; a < kDepthTile; ++a)
#pragma unroll
    for (int c = 0; c < kDepthTile; ++c)
#pragma unroll
      for (int v = 0; v < KV; ++v) acc[a][c][v] = 0.f;
  const float* g_img = ddepth + (size_t)b * Hu * Wu;

  for (int p = warp; p < npix; p += kDepthWarps) {
    const int y = ylo + p / nx, x = xlo + p % nx;
    const float g = __ldg(g_img + (size_t)y * Wu + x);
    const SegTap ty = seg_tap(y, h, sy), tx = seg_tap(x, w, sx);
    const int ly0 = ty.i0 - i0 + 1, ly1 = ty.i1 - i0 + 1, lx0 = tx.i0 - j0 + 1, lx1 = tx.i1 - j0 + 1;
    float r[KV], a[KV], S;
    const float d = depth_pixel<KV>(ty, tx, depth_sm + (ly0 * kDepthNb + lx0) * K, depth_sm + (ly0 * kDepthNb + lx1) * K,
                                    depth_sm + (ly1 * kDepthNb + lx0) * K, depth_sm + (ly1 * kDepthNb + lx1) * K, binv, K,
                                    lane, r, a, S);
    const float gs = g / S;
    float wgt[kDepthTile][kDepthTile];
#pragma unroll
    for (int ai = 0; ai < kDepthTile; ++ai) {
      const float wy = (ty.i0 == i0 + ai ? ty.l0 : 0.f) + (ty.i1 == i0 + ai ? ty.l1 : 0.f);
#pragma unroll
      for (int c = 0; c < kDepthTile; ++c) {
        const float wx = (tx.i0 == j0 + c ? tx.l0 : 0.f) + (tx.i1 == j0 + c ? tx.l1 : 0.f);
        wgt[ai][c] = wy * wx;
      }
    }
#pragma unroll
    for (int v = 0; v < KV; ++v) {
      const float dr = r[v] > 0.f ? gs * (binv[v] - d) : 0.f;
#pragma unroll
      for (int ai = 0; ai < kDepthTile; ++ai)
#pragma unroll
        for (int c = 0; c < kDepthTile; ++c) acc[ai][c][v] = fmaf(wgt[ai][c], dr, acc[ai][c][v]);
    }
  }
  __syncthreads();  // the neighbourhood is dead: reuse its shared memory for the per-warp sums
  float* red = depth_sm;
#pragma unroll
  for (int ai = 0; ai < kDepthTile; ++ai)
#pragma unroll
    for (int c = 0; c < kDepthTile; ++c)
#pragma unroll
      for (int v = 0; v < KV; ++v) {
        const int k = lane + 32 * v;
        if (k < K) red[((warp * kDepthTile + ai) * kDepthTile + c) * K + k] = acc[ai][c][v];
      }
  __syncthreads();
  for (int e = threadIdx.x; e < kDepthTile * kDepthTile * K; e += blockDim.x) {
    const int k = e % K, cell = e / K;
    const int i = i0 + cell / kDepthTile, j = j0 + cell % kDepthTile;
    if (i >= h || j >= w) continue;
    float sum = 0.f;
    for (int q = 0; q < kDepthWarps; ++q) sum += red[(q * kDepthTile * kDepthTile + cell) * K + k];
    dlogits[(((size_t)b * h + i) * w + j) * K + k] = sum;
  }
}

#define DVT_DEPTH_KV_DISPATCH(KVAR, MACRO) \
  do {                                     \
    if ((KVAR) <= 1) MACRO(1);             \
    else if ((KVAR) <= 2) MACRO(2);        \
    else if ((KVAR) <= 4) MACRO(4);        \
    else MACRO(8);                         \
  } while (0)

static int depth_head_check(const char* what, const float* a, const float* bins, const float* c, int B, int h, int w, int K,
                            int up) {
  DVT_REQUIRE(a && bins && c, "%s: null argument", what);
  DVT_REQUIRE(B > 0 && h > 0 && w > 0 && up > 0, "%s: bad shape B=%d h=%d w=%d upsample=%d", what, B, h, w, up);
  DVT_REQUIRE((long long)h * up < (1 << 20) && (long long)w * up < (1 << 20), "%s: %dx%d x%d is too large", what, h, w, up);
  DVT_REQUIRE(K >= 1 && K <= 256, "%s: n_bins=%d unsupported (1..256)", what, K);
  return DVT_OK;
}

int launch_depth_head_fwd(const float* logits, int B, int h, int w, int K, int up, const float* bins, float* depth,
                          cudaStream_t st) {
  const int rc = depth_head_check("depth_head_fwd", logits, bins, depth, B, h, w, K, up);
  if (rc != DVT_OK) return rc;
  const long long n = (long long)B * h * up * w * up;
  const int blocks = (int)std::min<long long>((n + kDepthWarps - 1) / kDepthWarps, (long long)num_sms() * 16);
  const int kv = (K + 31) / 32;
#define DVT_DEPTH_FWD(KV) depth_head_fwd_kernel<KV><<<blocks, kDepthWarps * 32, 0, st>>>(logits, B, h, w, K, up, bins, depth)
  DVT_DEPTH_KV_DISPATCH(kv, DVT_DEPTH_FWD);
#undef DVT_DEPTH_FWD
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

int launch_depth_head_bwd(const float* logits, int B, int h, int w, int K, int up, const float* bins, const float* ddepth,
                          float* dlogits, cudaStream_t st) {
  int rc = depth_head_check("depth_head_bwd", logits, bins, dlogits, B, h, w, K, up);
  if (rc != DVT_OK) return rc;
  DVT_REQUIRE(ddepth, "depth_head_bwd: null argument");
  const dim3 grid((w + kDepthTile - 1) / kDepthTile, (h + kDepthTile - 1) / kDepthTile, B);
  DVT_REQUIRE(B <= 65535 && grid.y <= 65535, "depth_head_bwd: B=%d h=%d exceed the grid", B, h);
  const size_t smem = (size_t)std::max(kDepthNb * kDepthNb, kDepthWarps * kDepthTile * kDepthTile) * K * sizeof(float);
  const int kv = (K + 31) / 32;
#define DVT_DEPTH_BWD(KV)                                                                                                   \
  do {                                                                                                                      \
    if (smem > 48 * 1024)                                                                                                   \
      DVT_CUDA_OK(cudaFuncSetAttribute(depth_head_bwd_kernel<KV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    depth_head_bwd_kernel<KV><<<grid, kDepthWarps * 32, smem, st>>>(logits, h, w, K, up, bins, ddepth, dlogits);            \
  } while (0)
  DVT_DEPTH_KV_DISPATCH(kv, DVT_DEPTH_BWD);
#undef DVT_DEPTH_BWD
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// One-channel bilinear resize [B, Hi, Wi] -> [B, Ho, Wo]: forward one thread per output pixel; backward one thread per
// input cell, gathering over the output pixels whose taps reach it (rows, then columns, ascending).  The candidate
// window is widened by 2 on each side of the analytic bound and every candidate is tested with the exact tap, so the
// gather equals the scatter of F.interpolate's backward up to the order of the adds.
// ----------------------------------------------------------------------------------------------------
__global__ void depth_resize_fwd_kernel(const float* __restrict__ in, int B, int Hi, int Wi, float* __restrict__ out, int Ho,
                                        int Wo) {
  const float sy = (float)Hi / (float)Ho, sx = (float)Wi / (float)Wo;
  const long long n = (long long)B * Ho * Wo;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(e / ((long long)Ho * Wo));
    const int p = (int)(e % ((long long)Ho * Wo));
    const SegTap ty = seg_tap(p / Wo, Hi, sy), tx = seg_tap(p % Wo, Wi, sx);
    const float* v = in + (size_t)b * Hi * Wi;
    out[e] = seg_lerp(ty, tx, __ldg(v + (size_t)ty.i0 * Wi + tx.i0), __ldg(v + (size_t)ty.i0 * Wi + tx.i1),
                      __ldg(v + (size_t)ty.i1 * Wi + tx.i0), __ldg(v + (size_t)ty.i1 * Wi + tx.i1));
  }
}

__device__ __forceinline__ void depth_gather_range(int i, int in_size, int out_size, float scale, int& lo, int& hi) {
  // i0(d) lies in {i - 1, i} only if src(d) = scale (d + 0.5) - 0.5 lies in [i - 1, i + 1)
  lo = max((int)floorf(((float)i - 0.5f) / scale - 0.5f) - 2, 0);
  hi = min((int)ceilf(((float)i + 1.5f) / scale - 0.5f) + 2, out_size - 1);
}

__global__ void depth_resize_bwd_kernel(const float* __restrict__ dout, int B, int Hi, int Wi, int Ho, int Wo,
                                        float* __restrict__ din) {
  const float sy = (float)Hi / (float)Ho, sx = (float)Wi / (float)Wo;
  const long long n = (long long)B * Hi * Wi;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(e / ((long long)Hi * Wi));
    const int p = (int)(e % ((long long)Hi * Wi));
    const int i = p / Wi, j = p % Wi;
    int ylo, yhi, xlo, xhi;
    depth_gather_range(i, Hi, Ho, sy, ylo, yhi);
    depth_gather_range(j, Wi, Wo, sx, xlo, xhi);
    const float* g = dout + (size_t)b * Ho * Wo;
    float sum = 0.f;
    for (int y = ylo; y <= yhi; ++y) {
      const SegTap ty = seg_tap(y, Hi, sy);
      if (ty.i0 != i && ty.i1 != i) continue;
      const float wy = (ty.i0 == i ? ty.l0 : 0.f) + (ty.i1 == i ? ty.l1 : 0.f);
      for (int x = xlo; x <= xhi; ++x) {
        const SegTap tx = seg_tap(x, Wi, sx);
        if (tx.i0 != j && tx.i1 != j) continue;
        const float wx = (tx.i0 == j ? tx.l0 : 0.f) + (tx.i1 == j ? tx.l1 : 0.f);
        sum = fmaf(wy * wx, __ldg(g + (size_t)y * Wo + x), sum);
      }
    }
    din[e] = sum;
  }
}

static int depth_resize_check(const char* what, const float* a, const float* c, int B, int Hi, int Wi, int Ho, int Wo) {
  DVT_REQUIRE(a && c, "%s: null argument", what);
  DVT_REQUIRE(B > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0, "%s: bad shape B=%d %dx%d -> %dx%d", what, B, Hi, Wi, Ho, Wo);
  return DVT_OK;
}

int launch_depth_resize_fwd(const float* in, int B, int Hi, int Wi, float* out, int Ho, int Wo, cudaStream_t st) {
  const int rc = depth_resize_check("depth_resize_fwd", in, out, B, Hi, Wi, Ho, Wo);
  if (rc != DVT_OK) return rc;
  const long long n = (long long)B * Ho * Wo;
  const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)num_sms() * 8);
  depth_resize_fwd_kernel<<<blocks, 256, 0, st>>>(in, B, Hi, Wi, out, Ho, Wo);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

int launch_depth_resize_bwd(const float* dout, int B, int Hi, int Wi, int Ho, int Wo, float* din, cudaStream_t st) {
  const int rc = depth_resize_check("depth_resize_bwd", dout, din, B, Hi, Wi, Ho, Wo);
  if (rc != DVT_OK) return rc;
  const long long n = (long long)B * Hi * Wi;
  const int blocks = (int)std::min<long long>((n + 255) / 256, (long long)num_sms() * 8);
  depth_resize_bwd_kernel<<<blocks, 256, 0, st>>>(dout, B, Hi, Wi, Ho, Wo, din);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Whole-image evaluation of one image with test-time augmentation: for every pixel of the original Ho x Wo image, the
// bilinear taps of each augmentation's Hu x Wu map clamped to [min_depth, max_depth] (the clamp of the reference's
// encode_decode, made before its resize; clamping the four taps is the same), a flipped augmentation read at column
// Wo - 1 - x, the augmentations added in order and divided by their number in fp32, then the masks (min < gt < max and
// the crop box) and the f64 per-pixel terms of the reference's calculate():
//   [count, ratio < 1.25, < 1.25^2, < 1.25^3 (ratio max(gt/pred, pred/gt) in fp32), sum |d|/gt, sum d^2/gt, sum d^2,
//    sum err, sum err^2, sum |log10 gt - log10 pred|], d = gt - pred, err = log pred - log gt.
// (log gt - log pred)^2 of rmse_log is err^2.  Each CTA reduces its pixels in a fixed order (thread, then warp
// butterfly, then warps in order) into part[blk][10]; depth_eval_final_kernel adds the kDepthEvalBlocks partials in order.
// ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kDepthEvalThreads) depth_eval_kernel(const float* __restrict__ maps, int n_aug,
                                                                       unsigned int flip_mask, int Hu, int Wu,
                                                                       const float* __restrict__ gt, int Ho, int Wo,
                                                                       float min_depth, float max_depth, int cy0, int cy1,
                                                                       int cx0, int cx1, double* __restrict__ part) {
  __shared__ double s_red[kDepthEvalThreads / 32][kDepthSums];
  const float sy = (float)Hu / (float)Ho, sx = (float)Wu / (float)Wo;
  const size_t plane = (size_t)Hu * Wu;
  double acc[kDepthSums];
#pragma unroll
  for (int s = 0; s < kDepthSums; ++s) acc[s] = 0.0;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Ho * Wo; e += gridDim.x * blockDim.x) {
    const int y = e / Wo, x = e % Wo;
    const float g = __ldg(gt + e);
    if (!(g > min_depth && g < max_depth) || y < cy0 || y >= cy1 || x < cx0 || x >= cx1) continue;
    const SegTap ty = seg_tap(y, Hu, sy);
    float sum = 0.f;
    for (int a = 0; a < n_aug; ++a) {
      const SegTap tx = seg_tap((flip_mask >> a) & 1u ? Wo - 1 - x : x, Wu, sx);
      const float* m = maps + a * plane;
      const float v00 = fminf(fmaxf(__ldg(m + (size_t)ty.i0 * Wu + tx.i0), min_depth), max_depth);
      const float v01 = fminf(fmaxf(__ldg(m + (size_t)ty.i0 * Wu + tx.i1), min_depth), max_depth);
      const float v10 = fminf(fmaxf(__ldg(m + (size_t)ty.i1 * Wu + tx.i0), min_depth), max_depth);
      const float v11 = fminf(fmaxf(__ldg(m + (size_t)ty.i1 * Wu + tx.i1), min_depth), max_depth);
      sum += seg_lerp(ty, tx, v00, v01, v10, v11);
    }
    const float p = sum / (float)n_aug;
    const float ratio = fmaxf(g / p, p / g);
    const double gd = g, pd = p, d = gd - pd, err = log(pd) - log(gd);
    acc[0] += 1.0;
    acc[1] += ratio < 1.25f ? 1.0 : 0.0;
    acc[2] += ratio < 1.5625f ? 1.0 : 0.0;
    acc[3] += ratio < 1.953125f ? 1.0 : 0.0;
    acc[4] += fabs(d) / gd;
    acc[5] += d * d / gd;
    acc[6] += d * d;
    acc[7] += err;
    acc[8] += err * err;
    acc[9] += fabs(log10(gd) - log10(pd));
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int s = 0; s < kDepthSums; ++s) {
    const double v = warp_sum_d(acc[s]);
    if (lane == 0) s_red[warp][s] = v;
  }
  __syncthreads();
  if (threadIdx.x < kDepthSums) {
    double v = 0.0;
    for (int q = 0; q < kDepthEvalThreads / 32; ++q) v += s_red[q][threadIdx.x];
    part[(size_t)blockIdx.x * kDepthSums + threadIdx.x] = v;
  }
}

__global__ void depth_eval_final_kernel(const double* __restrict__ part, int nblk, double* __restrict__ sums) {
  if (threadIdx.x < kDepthSums) {
    double v = 0.0;
    for (int q = 0; q < nblk; ++q) v += part[(size_t)q * kDepthSums + threadIdx.x];
    sums[threadIdx.x] = v;
  }
}

int launch_depth_eval_sums(const float* maps, int n_aug, unsigned int flip_mask, int Hu, int Wu, const float* gt, int Ho,
                           int Wo, float min_depth, float max_depth, int cy0, int cy1, int cx0, int cx1, double* workspace,
                           double* sums, cudaStream_t st) {
  DVT_REQUIRE(maps && gt && workspace && sums, "depth_eval_sums: null argument");
  DVT_REQUIRE(n_aug >= 1 && n_aug <= 32 && Hu > 0 && Wu > 0 && Ho > 0 && Wo > 0,
              "depth_eval_sums: bad shape n_aug=%d map %dx%d image %dx%d", n_aug, Hu, Wu, Ho, Wo);
  DVT_REQUIRE(min_depth < max_depth, "depth_eval_sums: min_depth %g >= max_depth %g", (double)min_depth, (double)max_depth);
  depth_eval_kernel<<<kDepthEvalBlocks, kDepthEvalThreads, 0, st>>>(maps, n_aug, flip_mask, Hu, Wu, gt, Ho, Wo, min_depth,
                                                                    max_depth, cy0, cy1, cx0, cx1, workspace);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  depth_eval_final_kernel<<<1, 32, 0, st>>>(workspace, kDepthEvalBlocks, sums);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

#undef DVT_DEPTH_KV_DISPATCH

}  // namespace dvt
