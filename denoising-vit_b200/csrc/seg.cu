// Dense-task linear probe (semantic segmentation): the full-resolution parts of the training loss and of slide inference.
//
// Every kernel here reproduces ATen's upsample_bilinear2d with align_corners=False in fp32: along an axis of `in` source
// cells resized to `out` pixels, scale = (float)in / out, src = max(scale * (dst + 0.5) - 0.5, 0), i0 = (int)src,
// i1 = i0 + (i0 < in - 1), weights (1 - (src - i0), src - i0), and the value
//   l0y * (l0x * v[i0y, i0x] + l1x * v[i0y, i1x]) + l1y * (l0x * v[i1y, i0x] + l1x * v[i1y, i1x]).
// No float atomics: every sum has a fixed order, so repeated calls are bit-identical.
#include "common.cuh"

#include <algorithm>

namespace dvt {

namespace {

struct SegTap {
  int i0, i1;
  float l0, l1;
};

__device__ __forceinline__ SegTap seg_tap(int dst, int in_size, float scale) {
  float src = scale * ((float)dst + 0.5f) - 0.5f;
  src = src < 0.f ? 0.f : src;
  SegTap t;
  t.i0 = (int)src;
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  t.l1 = src - (float)t.i0;
  t.l0 = 1.f - t.l1;
  return t;
}

__device__ __forceinline__ float seg_lerp(const SegTap& ty, const SegTap& tx, float v00, float v01, float v10, float v11) {
  return ty.l0 * (tx.l0 * v00 + tx.l1 * v01) + ty.l1 * (tx.l0 * v10 + tx.l1 * v11);
}

__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

constexpr int kSegTile = 2;     // low-resolution cells per CTA along each axis
constexpr int kSegWarps = 8;
constexpr int kSegNb = kSegTile + 2;

}  // namespace

// ----------------------------------------------------------------------------------------------------
// Fused bilinear upsample + softmax cross-entropy + gradient, gathered back to the low resolution.
// CTA = (2 x 2 low-resolution cells, image).  It walks every label pixel whose 4-tap footprint touches one of its cells
// (one warp per pixel, lanes over the classes k = lane + 32 kv), recomputes the pixel's K logits from the 4 x 4
// neighbourhood of cells staged in shared memory, and adds w * dCE/dlogit into per-warp register accumulators of its
// cells.  The warps' accumulators are then added in warp order.  A pixel's loss is counted by the CTA that owns its top-left
// tap; per-CTA loss partials (f64) go to `part` and are added in a fixed order by seg_loss_final_kernel.
// ----------------------------------------------------------------------------------------------------
template <int KV>
__global__ void __launch_bounds__(kSegWarps * 32) seg_upsample_ce_kernel(
    const float* __restrict__ logits, int h, int w, int K, const uint8_t* __restrict__ labels, int H, int W,
    float grad_scale, float* __restrict__ dlogits, double* __restrict__ part) {
  extern __shared__ float seg_sm[];  // [nb cells][K] neighbourhood, later [warps][tile cells][K] partial sums
  __shared__ int s_lo[2], s_hi[2];
  __shared__ double s_loss[kSegWarps];
  const int b = blockIdx.z, i0 = blockIdx.y * kSegTile, j0 = blockIdx.x * kSegTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float sy = (float)h / (float)H, sx = (float)w / (float)W;
  if (threadIdx.x < 2) {
    s_lo[threadIdx.x] = 1 << 30;
    s_hi[threadIdx.x] = -1;
  }
  // neighbourhood: cell rows i0-1 .. i0+tile, cols j0-1 .. j0+tile (those inside the grid)
  const float* src = logits + (size_t)b * h * w * K;
  for (int e = threadIdx.x; e < kSegNb * kSegNb * K; e += blockDim.x) {
    const int k = e % K, c = e / K;
    const int r = i0 - 1 + c / kSegNb, q = j0 - 1 + c % kSegNb;
    if (r >= 0 && r < h && q >= 0 && q < w) seg_sm[e] = __ldg(src + ((size_t)r * w + q) * K + k);
  }
  __syncthreads();
  // pixel rows (columns) whose top tap lies in [i0 - 1, i0 + tile - 1]: exactly those that reach a cell of the tile
  for (int y = threadIdx.x; y < H; y += blockDim.x) {
    const int r = seg_tap(y, h, sy).i0;
    if (r >= i0 - 1 && r <= i0 + kSegTile - 1) {
      atomicMin(&s_lo[0], y);
      atomicMax(&s_hi[0], y);
    }
  }
  for (int x = threadIdx.x; x < W; x += blockDim.x) {
    const int q = seg_tap(x, w, sx).i0;
    if (q >= j0 - 1 && q <= j0 + kSegTile - 1) {
      atomicMin(&s_lo[1], x);
      atomicMax(&s_hi[1], x);
    }
  }
  __syncthreads();
  const int ylo = s_lo[0], xlo = s_lo[1];
  const int ny = s_hi[0] - ylo + 1, nx = s_hi[1] - xlo + 1;
  const int npix = (ny > 0 && nx > 0) ? ny * nx : 0;

  float acc[kSegTile][kSegTile][KV];
#pragma unroll
  for (int a = 0; a < kSegTile; ++a)
#pragma unroll
    for (int c = 0; c < kSegTile; ++c)
#pragma unroll
      for (int v = 0; v < KV; ++v) acc[a][c][v] = 0.f;
  double loss = 0.0;
  const uint8_t* lab_img = labels + (size_t)b * H * W;

  for (int p = warp; p < npix; p += kSegWarps) {
    const int y = ylo + p / nx, x = xlo + p % nx;
    const int lab = lab_img[(size_t)y * W + x];
    if (lab >= K) continue;  // 255 (ignore): no loss, zero gradient
    const SegTap ty = seg_tap(y, h, sy), tx = seg_tap(x, w, sx);
    const int ly0 = ty.i0 - i0 + 1, ly1 = ty.i1 - i0 + 1, lx0 = tx.i0 - j0 + 1, lx1 = tx.i1 - j0 + 1;
    const float* c00 = seg_sm + (ly0 * kSegNb + lx0) * K;
    const float* c01 = seg_sm + (ly0 * kSegNb + lx1) * K;
    const float* c10 = seg_sm + (ly1 * kSegNb + lx0) * K;
    const float* c11 = seg_sm + (ly1 * kSegNb + lx1) * K;
    float val[KV];
    float m = -INFINITY, zlab = 0.f;
#pragma unroll
    for (int v = 0; v < KV; ++v) {
      const int k = lane + 32 * v;
      val[v] = k < K ? seg_lerp(ty, tx, c00[k], c01[k], c10[k], c11[k]) : -INFINITY;
      m = fmaxf(m, val[v]);
      if (k == lab) zlab = val[v];
    }
    m = warp_max_f(m);
    zlab = __shfl_sync(0xffffffffu, zlab, lab & 31);
    float s = 0.f;
#pragma unroll
    for (int v = 0; v < KV; ++v) {
      val[v] = expf(val[v] - m);  // exp(-inf) = 0 for the padding lanes
      s += val[v];
    }
    s = warp_sum_f(s);
    const bool owner = ty.i0 >= i0 && ty.i0 < i0 + kSegTile && tx.i0 >= j0 && tx.i0 < j0 + kSegTile;
    if (owner && lane == 0) loss += (double)(m + logf(s) - zlab);   // lse - z_lab
    const float inv = 1.f / s;
    float wgt[kSegTile][kSegTile];
#pragma unroll
    for (int a = 0; a < kSegTile; ++a) {
      const float wy = (ty.i0 == i0 + a ? ty.l0 : 0.f) + (ty.i1 == i0 + a ? ty.l1 : 0.f);
#pragma unroll
      for (int c = 0; c < kSegTile; ++c) {
        const float wx = (tx.i0 == j0 + c ? tx.l0 : 0.f) + (tx.i1 == j0 + c ? tx.l1 : 0.f);
        wgt[a][c] = wy * wx;
      }
    }
#pragma unroll
    for (int v = 0; v < KV; ++v) {
      const int k = lane + 32 * v;
      const float g = (val[v] * inv - (k == lab ? 1.f : 0.f)) * grad_scale;
#pragma unroll
      for (int a = 0; a < kSegTile; ++a)
#pragma unroll
        for (int c = 0; c < kSegTile; ++c) acc[a][c][v] = fmaf(wgt[a][c], g, acc[a][c][v]);
    }
  }
  __syncthreads();  // the neighbourhood is dead: reuse its shared memory for the per-warp sums
  float* red = seg_sm;
#pragma unroll
  for (int a = 0; a < kSegTile; ++a)
#pragma unroll
    for (int c = 0; c < kSegTile; ++c)
#pragma unroll
      for (int v = 0; v < KV; ++v) {
        const int k = lane + 32 * v;
        if (k < K) red[((warp * kSegTile + a) * kSegTile + c) * K + k] = acc[a][c][v];
      }
  if (lane == 0) s_loss[warp] = loss;
  __syncthreads();
  for (int e = threadIdx.x; e < kSegTile * kSegTile * K; e += blockDim.x) {
    const int k = e % K, cell = e / K;
    const int i = i0 + cell / kSegTile, j = j0 + cell % kSegTile;
    if (i >= h || j >= w) continue;
    float sum = 0.f;
    for (int q = 0; q < kSegWarps; ++q) sum += red[(q * kSegTile * kSegTile + cell) * K + k];
    dlogits[(((size_t)b * h + i) * w + j) * K + k] = sum;
  }
  if (threadIdx.x == 0) {
    double l = 0.0;
    for (int q = 0; q < kSegWarps; ++q) l += s_loss[q];
    part[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = l;
  }
}

// One CTA of kSegFinalThreads: thread t adds partials t, t + T, t + 2T, ... in order, then a shared-memory tree with a
// fixed pairing.  The order depends only on n, so the result is bit-identical from call to call.
constexpr int kSegFinalThreads = 256;
__global__ void __launch_bounds__(kSegFinalThreads) seg_loss_final_kernel(const double* __restrict__ part, int n,
                                                                         float* __restrict__ loss_out) {
  __shared__ double s[kSegFinalThreads];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += kSegFinalThreads) acc += part[i];
  s[threadIdx.x] = acc;
  __syncthreads();
#pragma unroll
  for (int stride = kSegFinalThreads / 2; stride > 0; stride >>= 1) {
    if (threadIdx.x < stride) s[threadIdx.x] += s[threadIdx.x + stride];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss_out[0] = (float)s[0];
}

int launch_seg_upsample_ce(const float* logits, int B, int h, int w, int K, const uint8_t* labels, int H, int W,
                           float grad_scale, float* loss_out, float* dlogits, double* workspace, cudaStream_t st) {
  DVT_REQUIRE(logits && labels && loss_out && dlogits && workspace, "seg_upsample_ce: null argument");
  DVT_REQUIRE(B > 0 && h > 0 && w > 0 && H > 0 && W > 0, "seg_upsample_ce: bad shape B=%d h=%d w=%d H=%d W=%d", B, h, w, H, W);
  DVT_REQUIRE(K >= 2 && K <= 255, "seg_upsample_ce: K=%d unsupported (2..255 classes; label 255 is ignore)", K);
  const int kv = (K + 31) / 32;
  const dim3 grid((w + kSegTile - 1) / kSegTile, (h + kSegTile - 1) / kSegTile, B);
  const size_t smem = (size_t)std::max(kSegNb * kSegNb, kSegWarps * kSegTile * kSegTile) * K * sizeof(float);
#define DVT_SEG_CE(KV)                                                                                                   \
  do {                                                                                                                   \
    if (smem > 48 * 1024)                                                                                                \
      DVT_CUDA_OK(cudaFuncSetAttribute(seg_upsample_ce_kernel<KV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    seg_upsample_ce_kernel<KV><<<grid, kSegWarps * 32, smem, st>>>(logits, h, w, K, labels, H, W, grad_scale, dlogits,    \
                                                                   workspace);                                         \
  } while (0)
  if (kv <= 1) DVT_SEG_CE(1);
  else if (kv <= 2) DVT_SEG_CE(2);
  else if (kv <= 3) DVT_SEG_CE(3);
  else if (kv <= 5) DVT_SEG_CE(5);
  else DVT_SEG_CE(8);
#undef DVT_SEG_CE
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  seg_loss_final_kernel<<<1, kSegFinalThreads, 0, st>>>(workspace, (int)(grid.x * grid.y * grid.z), loss_out);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Slide inference, one window: acc[k, y1 + y, x1 + x] += upsample(logits)[y, x, k] for the window's wh x ww pixels, and
// count[y1 + y, x1 + x] += 1.  One thread per window pixel, classes in order; windows enqueued in order on one stream
// make every per-pixel sum follow that order.
// ----------------------------------------------------------------------------------------------------
__global__ void seg_slide_accumulate_kernel(const float* __restrict__ logits, int h, int w, int K, int y1, int x1, int wh,
                                            int ww, float* __restrict__ acc, float* __restrict__ count, int Hc, int Wc) {
  const float sy = (float)h / (float)wh, sx = (float)w / (float)ww;
  const size_t plane = (size_t)Hc * Wc;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < wh * ww; e += gridDim.x * blockDim.x) {
    const int y = e / ww, x = e % ww;
    const SegTap ty = seg_tap(y, h, sy), tx = seg_tap(x, w, sx);
    const float* c00 = logits + ((size_t)ty.i0 * w + tx.i0) * K;
    const float* c01 = logits + ((size_t)ty.i0 * w + tx.i1) * K;
    const float* c10 = logits + ((size_t)ty.i1 * w + tx.i0) * K;
    const float* c11 = logits + ((size_t)ty.i1 * w + tx.i1) * K;
    const size_t o = (size_t)(y1 + y) * Wc + (x1 + x);
    for (int k = 0; k < K; ++k)
      acc[(size_t)k * plane + o] += seg_lerp(ty, tx, __ldg(c00 + k), __ldg(c01 + k), __ldg(c10 + k), __ldg(c11 + k));
    count[o] += 1.f;
  }
}

int launch_seg_slide_accumulate(const float* logits, int h, int w, int K, int y1, int x1, int wh, int ww, float* acc,
                                float* count, int Hc, int Wc, cudaStream_t st) {
  DVT_REQUIRE(logits && acc && count, "seg_slide_accumulate: null argument");
  DVT_REQUIRE(h > 0 && w > 0 && K > 0 && wh > 0 && ww > 0, "seg_slide_accumulate: bad shape h=%d w=%d K=%d window %dx%d", h,
              w, K, wh, ww);
  DVT_REQUIRE(y1 >= 0 && x1 >= 0 && y1 + wh <= Hc && x1 + ww <= Wc,
              "seg_slide_accumulate: window (%d, %d) %dx%d outside the %dx%d accumulator", y1, x1, wh, ww, Hc, Wc);
  const int blocks = (int)std::min<long long>(((long long)wh * ww + 255) / 256, (long long)num_sms() * 8);
  seg_slide_accumulate_kernel<<<blocks, 256, 0, st>>>(logits, h, w, K, y1, x1, wh, ww, acc, count, Hc, Wc);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Slide inference, end of an image: acc /= count (in place, the division mmseg makes before resizing), then per pixel of
// the original image the bilinear resize from Hc x Wc to Ho x Wo, argmax over the classes (ties -> lowest index, as
// torch.argmax) and the per-class histograms of mmseg's intersect_and_union in shared memory, added to
// hist [4, K] = (intersect, union, pred, label) with integer atomics (exact, order-free).
// ----------------------------------------------------------------------------------------------------
__global__ void seg_divide_kernel(float* __restrict__ acc, const float* __restrict__ count, size_t plane, int K) {
  const size_t n = plane * K;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x)
    acc[e] = acc[e] / count[e % plane];
}

__global__ void seg_predict_hist_kernel(const float* __restrict__ mean, int K, int Hc, int Wc, const uint8_t* __restrict__ labels,
                                        int Ho, int Wo, unsigned long long* __restrict__ hist) {
  extern __shared__ unsigned int s_hist[];  // [3][K]: intersect, pred, label
  for (int e = threadIdx.x; e < 3 * K; e += blockDim.x) s_hist[e] = 0u;
  __syncthreads();
  const float sy = (float)Hc / (float)Ho, sx = (float)Wc / (float)Wo;
  const size_t plane = (size_t)Hc * Wc;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Ho * Wo; e += gridDim.x * blockDim.x) {
    const int lab = labels[e];
    if (lab == 255) continue;
    const int y = e / Wo, x = e % Wo;
    const SegTap ty = seg_tap(y, Hc, sy), tx = seg_tap(x, Wc, sx);
    const size_t o00 = (size_t)ty.i0 * Wc + tx.i0, o01 = (size_t)ty.i0 * Wc + tx.i1;
    const size_t o10 = (size_t)ty.i1 * Wc + tx.i0, o11 = (size_t)ty.i1 * Wc + tx.i1;
    float best = -INFINITY;
    int arg = 0;
    for (int k = 0; k < K; ++k) {
      const float* pk = mean + (size_t)k * plane;
      const float v = seg_lerp(ty, tx, __ldg(pk + o00), __ldg(pk + o01), __ldg(pk + o10), __ldg(pk + o11));
      if (v > best) {
        best = v;
        arg = k;
      }
    }
    atomicAdd(&s_hist[K + arg], 1u);
    if (lab < K) {
      atomicAdd(&s_hist[2 * K + lab], 1u);
      if (arg == lab) atomicAdd(&s_hist[lab], 1u);
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const unsigned int it = s_hist[k], pr = s_hist[K + k], lb = s_hist[2 * K + k];
    if (it) atomicAdd(hist + k, (unsigned long long)it);
    if (pr + lb - it) atomicAdd(hist + K + k, (unsigned long long)(pr + lb - it));
    if (pr) atomicAdd(hist + 2 * K + k, (unsigned long long)pr);
    if (lb) atomicAdd(hist + 3 * K + k, (unsigned long long)lb);
  }
}

int launch_seg_predict_hist(float* acc, const float* count, int K, int Hc, int Wc, const uint8_t* labels, int Ho, int Wo,
                            unsigned long long* hist, cudaStream_t st) {
  DVT_REQUIRE(acc && count && labels && hist, "seg_predict_hist: null argument");
  DVT_REQUIRE(K > 0 && K <= 255 && Hc > 0 && Wc > 0 && Ho > 0 && Wo > 0,
              "seg_predict_hist: bad shape K=%d accumulator %dx%d image %dx%d", K, Hc, Wc, Ho, Wo);
  const size_t plane = (size_t)Hc * Wc;
  const int dblocks = (int)std::min<size_t>((plane * K + 255) / 256, (size_t)num_sms() * 8);
  seg_divide_kernel<<<dblocks, 256, 0, st>>>(acc, count, plane, K);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  const int blocks = (int)std::min<long long>(((long long)Ho * Wo + 255) / 256, (long long)num_sms() * 4);
  seg_predict_hist_kernel<<<blocks, 256, 3 * K * sizeof(unsigned int), st>>>(acc, K, Hc, Wc, labels, Ho, Wo, hist);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Test-time augmentation (mmseg EncoderDecoder.aug_test), one augmentation: for every pixel of the original Ho x Wo image
// the bilinear resize of acc / count from the augmentation's Hc x Wc (each tap divided by its count: the values of
// mmseg's preds / count_mat), the softmax over the classes, the horizontal un-flip of a flipped augmentation, and
// prob[k, y, x] += p_k.  A CTA takes kAugTile consecutive pixels at a time: one warp per pixel, lanes over the classes
// (k = lane + 32 v), probabilities staged in shared memory as [class][pixel], then added to prob by rows of kAugTile
// pixels per class (coalesced, where a warp's lanes over the classes would touch 32 planes).  A pixel is owned by one
// CTA, so augmentations enqueued in order on one stream add in that order.
// ----------------------------------------------------------------------------------------------------
constexpr int kAugTile = 32;

template <int KV>
__global__ void __launch_bounds__(kSegWarps * 32) seg_aug_accumulate_kernel(
    const float* __restrict__ acc, const float* __restrict__ count, int K, int Hc, int Wc, int flip,
    float* __restrict__ prob, int Ho, int Wo) {
  __shared__ float tile[KV * 32][kAugTile + 1];  // +1: a warp stores one pixel's classes down a column
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float sy = (float)Hc / (float)Ho, sx = (float)Wc / (float)Wo;
  const size_t plane = (size_t)Hc * Wc, oplane = (size_t)Ho * Wo;
  const int n = Ho * Wo;
  for (int t0 = blockIdx.x * kAugTile; t0 < n; t0 += gridDim.x * kAugTile) {
    for (int j = warp; j < kAugTile && t0 + j < n; j += kSegWarps) {
      const int e = t0 + j, y = e / Wo, x = e % Wo;
      // output column x of a flipped augmentation is column Wo - 1 - x of its resized map
      const SegTap ty = seg_tap(y, Hc, sy), tx = seg_tap(flip ? Wo - 1 - x : x, Wc, sx);
      const size_t o00 = (size_t)ty.i0 * Wc + tx.i0, o01 = (size_t)ty.i0 * Wc + tx.i1;
      const size_t o10 = (size_t)ty.i1 * Wc + tx.i0, o11 = (size_t)ty.i1 * Wc + tx.i1;
      const float n00 = __ldg(count + o00), n01 = __ldg(count + o01), n10 = __ldg(count + o10), n11 = __ldg(count + o11);
      float val[KV];
      float m = -INFINITY;
#pragma unroll
      for (int v = 0; v < KV; ++v) {
        const int k = lane + 32 * v;
        if (k < K) {
          const float* pk = acc + (size_t)k * plane;
          val[v] = seg_lerp(ty, tx, __ldg(pk + o00) / n00, __ldg(pk + o01) / n01, __ldg(pk + o10) / n10,
                            __ldg(pk + o11) / n11);
        } else {
          val[v] = -INFINITY;
        }
        m = fmaxf(m, val[v]);
      }
      m = warp_max_f(m);
      float s = 0.f;
#pragma unroll
      for (int v = 0; v < KV; ++v) {
        val[v] = expf(val[v] - m);  // exp(-inf) = 0 for the padding lanes
        s += val[v];
      }
      s = warp_sum_f(s);
#pragma unroll
      for (int v = 0; v < KV; ++v) tile[lane + 32 * v][j] = val[v] / s;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < K * kAugTile; i += blockDim.x) {
      const int k = i / kAugTile, j = i % kAugTile;
      if (t0 + j < n) prob[(size_t)k * oplane + t0 + j] += tile[k][j];
    }
    __syncthreads();
  }
}

int launch_seg_aug_accumulate(const float* acc, const float* count, int K, int Hc, int Wc, int flip, float* prob, int Ho,
                              int Wo, cudaStream_t st) {
  DVT_REQUIRE(acc && count && prob, "seg_aug_accumulate: null argument");
  DVT_REQUIRE(K > 0 && K <= 255 && Hc > 0 && Wc > 0 && Ho > 0 && Wo > 0,
              "seg_aug_accumulate: bad shape K=%d accumulator %dx%d image %dx%d", K, Hc, Wc, Ho, Wo);
  const int kv = (K + 31) / 32;
  const int blocks = (int)std::min<long long>(((long long)Ho * Wo + kAugTile - 1) / kAugTile, (long long)num_sms() * 8);
#define DVT_SEG_AUG(KV) \
  seg_aug_accumulate_kernel<KV><<<blocks, kSegWarps * 32, 0, st>>>(acc, count, K, Hc, Wc, flip ? 1 : 0, prob, Ho, Wo)
  if (kv <= 1) DVT_SEG_AUG(1);
  else if (kv <= 2) DVT_SEG_AUG(2);
  else if (kv <= 3) DVT_SEG_AUG(3);
  else if (kv <= 5) DVT_SEG_AUG(5);
  else DVT_SEG_AUG(8);
#undef DVT_SEG_AUG
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Test-time augmentation, end of an image: prob / n_aug (the division of mmseg's aug_test, made before the argmax),
// argmax over the classes (ties -> lowest index) and the histograms against the labels, in seg_predict_hist_kernel's
// scheme: [3][K] unsigned counters in shared memory, added to hist [4, K] = (intersect, union, pred, label) with integer
// atomics.
// ----------------------------------------------------------------------------------------------------
__global__ void seg_aug_argmax_hist_kernel(const float* __restrict__ prob, int n_aug, int K, const uint8_t* __restrict__ labels,
                                           int Ho, int Wo, unsigned long long* __restrict__ hist) {
  extern __shared__ unsigned int s_hist[];  // [3][K]: intersect, pred, label
  for (int e = threadIdx.x; e < 3 * K; e += blockDim.x) s_hist[e] = 0u;
  __syncthreads();
  const float n = (float)n_aug;
  const size_t plane = (size_t)Ho * Wo;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < Ho * Wo; e += gridDim.x * blockDim.x) {
    const int lab = labels[e];
    if (lab == 255) continue;
    float best = -INFINITY;
    int arg = 0;
    for (int k = 0; k < K; ++k) {
      const float v = __ldg(prob + (size_t)k * plane + e) / n;
      if (v > best) {
        best = v;
        arg = k;
      }
    }
    atomicAdd(&s_hist[K + arg], 1u);
    if (lab < K) {
      atomicAdd(&s_hist[2 * K + lab], 1u);
      if (arg == lab) atomicAdd(&s_hist[lab], 1u);
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const unsigned int it = s_hist[k], pr = s_hist[K + k], lb = s_hist[2 * K + k];
    if (it) atomicAdd(hist + k, (unsigned long long)it);
    if (pr + lb - it) atomicAdd(hist + K + k, (unsigned long long)(pr + lb - it));
    if (pr) atomicAdd(hist + 2 * K + k, (unsigned long long)pr);
    if (lb) atomicAdd(hist + 3 * K + k, (unsigned long long)lb);
  }
}

int launch_seg_aug_argmax_hist(const float* prob, int n_aug, int K, const uint8_t* labels, int Ho, int Wo,
                               unsigned long long* hist, cudaStream_t st) {
  DVT_REQUIRE(prob && labels && hist, "seg_aug_argmax_hist: null argument");
  DVT_REQUIRE(n_aug > 0 && K > 0 && K <= 255 && Ho > 0 && Wo > 0,
              "seg_aug_argmax_hist: bad shape n_aug=%d K=%d image %dx%d", n_aug, K, Ho, Wo);
  const int blocks = (int)std::min<long long>(((long long)Ho * Wo + 255) / 256, (long long)num_sms() * 4);
  seg_aug_argmax_hist_kernel<<<blocks, 256, 3 * K * sizeof(unsigned int), st>>>(prob, n_aug, K, labels, Ho, Wo, hist);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

}  // namespace dvt
