// HP-2: per-image neural-field denoiser fit (stage 1), no tiny-cuda-nn.
// Replaces the hot loop of `denoise_an_image` (main_img_denoising.py:67-89): SingleImageDenoiser.forward
// (dvt/models/offline_denoiser.py:92-140) + NeuralFeatureField (dvt/models/neural_feature_field.py:25-49, tcnn
// HashGrid + 2-layer MLP) + torch.optim.Adam with the reference's exact quirks (dense hash-grid gradient ->
// dense Adam sweep, loss scale never unscaled, per-parameter step counters, G frozen / residual MLP started after
// `freeze_step`; SURVEY.md section 8a).
//
// One step = a fixed set of kernels on five streams (captured into CUDA graphs of several steps by the host; the full
// schedule with its hazards is documented at fit_enqueue_step):
//   main  : GEMM h1 = relu(enc W1^T + b1), GEMM F = h1 W2^T + b2, loss (pred = F + G[r,c] (+R), MSE + cosine, d pred,
//           dG atomics, loss log), dgrad, dgrad, grid backward (vector atomics + touched-entry stamps),
//           encode of the NEXT step (hash-grid gather / interpolation with the pending Adam steps applied on the fly)
//   sides : gather of the sampled bank rows, residual MLP forward (3 GEMM) / backward (5 GEMM), weight-gradient GEMMs,
//           Adam(small params), and the dense Adam sweep of the hash table (one pass per window of k steps,
//           software-pipelined one to two windows deep)
// All GEMMs run on the tensor cores (gemm.cu) as 3xTF32 products of fp32 hi/lo planes (fp32-accurate: bf16 operands cannot
// hold the cosine >= 0.999 parity bar, see DESIGN.md); weight-gradient GEMMs read the activations as MN-major
// operands, so no transposed copies exist; bias gradients come from a ones column appended to the activation buffers.
//
// HBM layout: table p/m/v as two ping-pong copies of three fp32 arrays of n_entries*8, gradients as a ring of 2k
// such arrays with per-entry step stamps; "small" params (field MLP, G as [h*w, C],
// residual MLP) in one flat fp32 buffer with identically laid out m / v / grad buffers and TF32 hi/lo operand planes.
#include "common.cuh"
#include "gemm.cuh"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

namespace dvt {

constexpr int FIT_MAX_LEVELS = 16;
constexpr int FIT_F = 8;  // features per level
constexpr int FIT_MAX_WINDOW = 8;  // steps per pipelined table sweep (DVT_FIT_SWEEP_STEPS)

struct GridLevels {
  int n_levels;
  float scale[FIT_MAX_LEVELS];
  uint32_t res[FIT_MAX_LEVELS];
  uint32_t size[FIT_MAX_LEVELS];
  uint32_t offset[FIT_MAX_LEVELS + 1];
  uint32_t hashed[FIT_MAX_LEVELS];
};

// tcnn grid_index for 2-D inputs (oracle/hashgrid.py::corner_indices_weights restates the published algorithm)
__device__ __forceinline__ uint32_t grid_index(const GridLevels& g, int l, uint32_t x, uint32_t y) {
  uint32_t idx = g.hashed[l] ? (x ^ (y * 2654435761u)) : (x + y * g.res[l]);
  return idx % g.size[l];
}

struct CornerSet {
  uint32_t idx[4];
  float w[4];
};

__device__ __forceinline__ CornerSet grid_corners(const GridLevels& g, int l, float x, float y) {
  const float s = g.scale[l];
  float px = fmaf(s, x, 0.5f), py = fmaf(s, y, 0.5f);
  const float fx = floorf(px), fy = floorf(py);
  const uint32_t cx = (uint32_t)(int)fx, cy = (uint32_t)(int)fy;
  px -= fx;
  py -= fy;
  CornerSet c;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int dx = k & 1, dy = k >> 1;
    c.idx[k] = g.offset[l] + grid_index(g, l, cx + dx, cy + dy);
    c.w[k] = (dx ? px : 1.f - px) * (dy ? py : 1.f - py);
  }
  return c;
}

// The bank rows sampled at step s are idx_all[s * n .. s * n + n).  Inside a captured CUDA graph the step is not
// a launch-time constant, so kernels take (idx_all, step_base, step_off) and resolve s = *step_base + step_off on
// the device; idx_all == nullptr means "row i" (query mode).
// The bank / coordinate pointers of the current fit are read through a device-side record as well (FitInputs), so a
// captured graph stays valid when the next image's bank / sampling stream live in another buffer.
struct FitInputs {
  const float* bank;
  const float* coords;
  const int* idx;  // [num_iters + 1, bsz] sampling stream of the current fit (double-buffered by the host engine)
};
struct StepRows {
  const int* idx_all;
  const int* step_base;
  int step_off;
  const FitInputs* in;  // nullptr: the kernel's direct bank / coords argument is used (query mode, unit tests)
  __device__ __forceinline__ const float* coords(const float* direct) const { return in ? in->coords : direct; }
  __device__ __forceinline__ const float* bank(const float* direct) const { return in ? in->bank : direct; }
  __device__ __forceinline__ int step() const { return *step_base + step_off; }
  __device__ __forceinline__ const int* rows(int n) const {
    const int* base = in ? in->idx : idx_all;
    return base ? base + (size_t)step() * n : nullptr;
  }
};

// ----------------------------------------------------------------------------------------------------
// encode: one thread per (sample, level).
//
// "Peek" mode (software-pipelined Adam): the dense Adam sweep of step t runs CONCURRENTLY with the forward /
// backward of step t+1, so when step t+1 is encoded the table still holds the state of step t.  The encode kernel
// therefore applies Adam step t on the fly to the (few) entries it reads -- same adam1() arithmetic, same inputs, so
// the value is bit-identical to what the sweep stores later -- without writing anything back.
// ----------------------------------------------------------------------------------------------------
struct AdamScalars {
  float step_size, inv_bc2_sqrt;  // lr / (1 - b1^t),  1 / sqrt(1 - b2^t)
};

// Branch-free: one MUFU.SQRT and one MUFU.RCP per parameter (the IEEE sqrtf / division expand to ~40 instructions
// with slow-path branches, which made the sweep issue-bound instead of HBM-bound).
__device__ __forceinline__ void adam1(float& p, float& m, float& v, float g, float wd, float ss, float inv_bc2s) {
  g = fmaf(wd, p, g);
  m = fmaf(g - m, 0.1f, m);                 // lerp(m, g, 1 - beta1), beta1 = 0.9
  v = fmaf(v, 0.99f, 0.01f * g * g);        // beta2 = 0.99
  float sq;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(sq) : "f"(v));
  const float denom = fmaf(sq, inv_bc2s, 1e-15f);
  p = fmaf(-ss, __fdividef(m, denom), p);
}

// Optimiser state of the hash table.  The state S_b at the start of a sweep window lives in p/m/v[buf]: a window sweep
// reads buffer buf and writes the other one, so S_b stays readable while the sweep runs.  buf is the number of sweeps
// since fit_begin (step_base[1], advanced with the step counter) plus the sweeps enqueued before it in the same epoch,
// mod 2.  The gradient of step t is accumulated into ring slot t % ring; stamp[slot][entry] == t + 1 marks the entries
// it touched (the first touch of a step overwrites the slot's stale value, so no slot is ever re-zeroed).
struct TableBufs {
  float* p[2];
  float* m[2];
  float* v[2];
  float* g;          // [ring][n_entries * FIT_F]
  uint32_t* stamp;   // [ring][n_entries]
  int ring;
  size_t n_entries;
  __device__ __forceinline__ int slot(int step) const { return step % ring; }
  __device__ __forceinline__ float* g_of(int step) const { return g + (size_t)slot(step) * n_entries * FIT_F; }
  __device__ __forceinline__ uint32_t* stamp_of(int step) const { return stamp + (size_t)slot(step) * n_entries; }
};
#define DVT_SEL2(arr, i) ((i) ? (arr)[1] : (arr)[0])

__device__ __forceinline__ void adam8(float4& pa, float4& pb, float4& ma, float4& mb, float4& va, float4& vb,
                                      const float4& ga, const float4& gb, float wd, const AdamScalars s) {
  adam1(pa.x, ma.x, va.x, ga.x, wd, s.step_size, s.inv_bc2_sqrt);
  adam1(pa.y, ma.y, va.y, ga.y, wd, s.step_size, s.inv_bc2_sqrt);
  adam1(pa.z, ma.z, va.z, ga.z, wd, s.step_size, s.inv_bc2_sqrt);
  adam1(pa.w, ma.w, va.w, ga.w, wd, s.step_size, s.inv_bc2_sqrt);
  adam1(pb.x, mb.x, vb.x, gb.x, wd, s.step_size, s.inv_bc2_sqrt);
  adam1(pb.y, mb.y, vb.y, gb.y, wd, s.step_size, s.inv_bc2_sqrt);
  adam1(pb.z, mb.z, vb.z, gb.z, wd, s.step_size, s.inv_bc2_sqrt);
  adam1(pb.w, mb.w, vb.w, gb.w, wd, s.step_size, s.inv_bc2_sqrt);
}

// One thread per (sample, level, corner); the four corners of a cell sit in adjacent lanes and are combined with two
// shuffles.  npeek = number of Adam steps (0 .. MAXPEEK) that are still pending in the sweeps and are applied on the fly:
// the encoded step is s, the state that is read is S_{s - npeek}, in state buffer (step_base[1] + buf_off) & 1.  All
// stamp and gradient loads are issued before the first adam8 (the encode is on the critical path).
// table_fixed != nullptr: read that table (query mode).
template <int MAXPEEK>
__global__ void __launch_bounds__(256)
fit_encode_kernel(GridLevels g, TableBufs tb, const float* __restrict__ table_fixed, const float* __restrict__ coords,
                  StepRows sr, int n, float* __restrict__ enc, int ld_enc, size_t plane,
                  const AdamScalars* __restrict__ sc, float wd, int npeek, int buf_off) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int k = t & 3;
  // Threads past the end stay in the kernel (clamped to the last element, store predicated off): the shuffles below name
  // the full warp, and n * n_levels need not be a multiple of 8 (query mode: n = h * w).
  const bool live = (t >> 2) < n * g.n_levels;
  const int q = live ? (t >> 2) : n * g.n_levels - 1;
  pdl_wait();     // (no-ops unless launched with programmatic stream serialisation)
  pdl_trigger();
  const int i = q % n, l = q / n;
  const int* rows = sr.rows(n);
  const int r = rows ? rows[i] : i;
  const float2 xy = *reinterpret_cast<const float2*>(sr.coords(coords) + 2 * (size_t)r);
  // corner k of the cell (same arithmetic as grid_corners)
  const float s = g.scale[l];
  float px = fmaf(s, xy.x, 0.5f), py = fmaf(s, xy.y, 0.5f);
  const float fx = floorf(px), fy = floorf(py);
  const uint32_t cx = (uint32_t)(int)fx, cy = (uint32_t)(int)fy;
  px -= fx;
  py -= fy;
  const int dx = k & 1, dy = k >> 1;
  const size_t e = g.offset[l] + grid_index(g, l, cx + dx, cy + dy);
  const float w = (dx ? px : 1.f - px) * (dy ? py : 1.f - py);
  const int b = table_fixed ? 0 : sr.step() - npeek;  // state that is read
  const int buf = table_fixed ? 0 : (sr.step_base[1] + buf_off) & 1;
  const float* P = table_fixed ? table_fixed : DVT_SEL2(tb.p, buf);
  float4 pa = __ldcg(reinterpret_cast<const float4*>(P + e * FIT_F));
  float4 pb = __ldcg(reinterpret_cast<const float4*>(P + e * FIT_F) + 1);
  if (npeek > 0) {
    const float4* mp = reinterpret_cast<const float4*>(DVT_SEL2(tb.m, buf) + e * FIT_F);
    const float4* vp = reinterpret_cast<const float4*>(DVT_SEL2(tb.v, buf) + e * FIT_F);
    float4 ma = __ldcg(mp), mb = __ldcg(mp + 1), va = __ldcg(vp), vb = __ldcg(vp + 1);
    uint32_t st[MAXPEEK];
#pragma unroll
    for (int j = 0; j < MAXPEEK; ++j) st[j] = j < npeek ? __ldcg(tb.stamp_of(b + j) + e) : 0u;
    const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 ga[MAXPEEK], gb[MAXPEEK];
#pragma unroll
    for (int j = 0; j < MAXPEEK; ++j) {
      ga[j] = z4;
      gb[j] = z4;
      if (j < npeek && st[j] == (uint32_t)(b + j) + 1u) {
        const float4* gp = reinterpret_cast<const float4*>(tb.g_of(b + j) + e * FIT_F);
        ga[j] = __ldcg(gp);
        gb[j] = __ldcg(gp + 1);
      }
    }
#pragma unroll
    for (int j = 0; j < MAXPEEK; ++j)
      if (j < npeek) adam8(pa, pb, ma, mb, va, vb, ga[j], gb[j], wd, sc[b + j]);
  }
  float acc[FIT_F] = {w * pa.x, w * pa.y, w * pa.z, w * pa.w, w * pb.x, w * pb.y, w * pb.z, w * pb.w};
#pragma unroll
  for (int f = 0; f < FIT_F; ++f) {
    acc[f] += __shfl_xor_sync(0xffffffffu, acc[f], 1);
    acc[f] += __shfl_xor_sync(0xffffffffu, acc[f], 2);
  }
  // lane k stores one float4: k = 0/1 the hi plane (features 0-3 / 4-7), k = 2/3 the lo plane
  float o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float a = (k & 1) ? acc[4 + j] : acc[j];
    const float hi = tf32_hi(a);
    o[j] = (k & 2) ? a - hi : hi;
  }
  float* dst = enc + (size_t)i * ld_enc + l * FIT_F + (k & 1) * 4 + ((k & 2) ? plane : 0);
  if (live) *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
}

// fp32 encode (unit-test entry point: bit-level check of indices / weights against the oracle)
__global__ void fit_encode_f32_kernel(GridLevels g, const float* __restrict__ table, const float* __restrict__ coords,
                                      int n, float* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * g.n_levels) return;
  const int i = t % n, l = t / n;
  const float2 xy = *reinterpret_cast<const float2*>(coords + 2 * (size_t)i);
  const CornerSet c = grid_corners(g, l, xy.x, xy.y);
  for (int f = 0; f < FIT_F; ++f) {
    float a = 0.f;
    for (int k = 0; k < 4; ++k) a = fmaf(c.w[k], table[(size_t)c.idx[k] * FIT_F + f], a);
    out[(size_t)i * g.n_levels * FIT_F + l * FIT_F + f] = a;
  }
}

// corner indices + weights (unit-test entry point; "bit-exact patch indexing")
__global__ void fit_corners_kernel(GridLevels g, const float* __restrict__ coords, int n, uint32_t* __restrict__ idx,
                                   float* __restrict__ w) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * g.n_levels) return;
  const int i = t % n, l = t / n;
  const CornerSet c = grid_corners(g, l, coords[2 * i], coords[2 * i + 1]);
  for (int k = 0; k < 4; ++k) {
    idx[((size_t)i * g.n_levels + l) * 4 + k] = c.idx[k];
    w[((size_t)i * g.n_levels + l) * 4 + k] = c.w[k];
  }
}

// backward of the encoding: dense-table gradient accumulation, in a fixed order (the result does not depend on thread
// scheduling: float atomics would add the contributions of colliding samples in whatever order they arrive, and 2000 Adam
// steps turn that last-bit noise into visibly different fits).  CTA (level, part) owns the level's entries with
// entry % GB_PARTS == part; samples in chunks of GB_ROWS: the chunk's (entry, contribution) keys of this part are collected
// in shared memory and sorted (bitonic; the keys are unique, so the order is canonical), then the first thread of every run
// of equal entries sums the run in contribution order and adds it to the entry.
// `stamp` (optional): stamp[entry] = step + 1 marks the entries that received a gradient this step, so that the dense
// Adam sweep reads the gradient of touched entries only: 24 B/param of traffic instead of 32.  An entry whose stamp is
// not yet this step's holds a stale gradient of an earlier step: its first touch overwrites it (0 + contribution, the
// value an accumulation into a zeroed slot gives, signed zeros included) instead of adding to it.
// The gradient / stamp buffers form a ring (TableBufs): the backward of step t writes ring slot t % ring while the
// sweeps of the two windows before may still be reading theirs.  tb.stamp == nullptr: plain accumulation into tb.g
// (unit-test entry point).
constexpr int GB_ROWS = 2048;
constexpr int GB_N = 4 * GB_ROWS;                  // contributions per chunk (a power of two)
constexpr int GB_THREADS = 512;
constexpr int GB_PARTS = 8;                        // CTAs per level
constexpr int GB_SMEM = GB_N * (8 + 4);            // sort keys + corner weights
__global__ void __launch_bounds__(GB_THREADS, 1)
fit_grid_bwd_kernel(GridLevels g, const float* __restrict__ coords, StepRows sr, int n, const float* __restrict__ denc,
                    int ld_denc, TableBufs tb) {
  extern __shared__ unsigned long long gb_key[];   // [GB_N]: (entry within the level) << 32 | contribution
  float* gb_w = reinterpret_cast<float*>(gb_key + GB_N);  // [GB_N]: corner weight of each contribution
  __shared__ int gb_cnt;
  const int l = blockIdx.x;
  const uint32_t part = blockIdx.y;
  pdl_wait();     // (no-ops unless launched with programmatic stream serialisation)
  pdl_trigger();
  const int* rows = sr.rows(n);
  const float* xy_all = sr.coords(coords);
  const bool stamped = tb.stamp != nullptr;
  float* gtable = stamped ? tb.g_of(sr.step()) : tb.g;
  uint32_t* stamp = stamped ? tb.stamp_of(sr.step()) : nullptr;
  const uint32_t mark = stamped ? (uint32_t)sr.step() + 1u : 0u;
  const uint32_t base = g.offset[l];
  constexpr unsigned long long PAD = ~0ull;
  for (int r0 = 0; r0 < n; r0 += GB_ROWS) {
    const int cnt = min(GB_ROWS, n - r0);
    if (threadIdx.x == 0) gb_cnt = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += GB_THREADS) {
      const int r = rows ? rows[r0 + i] : r0 + i;
      const float2 xy = *reinterpret_cast<const float2*>(xy_all + 2 * (size_t)r);
      const CornerSet c = grid_corners(g, l, xy.x, xy.y);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t e = c.idx[k] - base;
        if (e % GB_PARTS != part) continue;
        gb_key[atomicAdd(&gb_cnt, 1)] = ((unsigned long long)e << 32) | (unsigned)(4 * i + k);
        gb_w[4 * i + k] = c.w[k];
      }
    }
    __syncthreads();
    const int m = gb_cnt;
    int np = 2;
    while (np < m) np <<= 1;
    for (int p = m + threadIdx.x; p < np; p += GB_THREADS) gb_key[p] = PAD;
    __syncthreads();
    for (int k = 2; k <= np; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int t = threadIdx.x; t < np / 2; t += GB_THREADS) {
          const int lo = 2 * t - (t & (j - 1)), hi = lo + j;  // pair t: index with a 0 inserted at bit log2(j), and its partner
          const unsigned long long x = gb_key[lo], y = gb_key[hi];
          if ((x > y) == ((lo & k) == 0)) {
            gb_key[lo] = y;
            gb_key[hi] = x;
          }
        }
        __syncthreads();
      }
    }
    for (int p = threadIdx.x; p < m; p += GB_THREADS) {
      const uint32_t e = (uint32_t)(gb_key[p] >> 32);
      if (p > 0 && (uint32_t)(gb_key[p - 1] >> 32) == e) continue;  // not the first of its run
      float4 sa = make_float4(0.f, 0.f, 0.f, 0.f), sb = sa;
      for (int q = p; q < m && (uint32_t)(gb_key[q] >> 32) == e; ++q) {
        const uint32_t ci = (uint32_t)gb_key[q];
        const float w = gb_w[ci];
        const float* src = denc + (size_t)(r0 + (ci >> 2)) * ld_denc + l * FIT_F;
        const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
        sa.x += w * a.x; sa.y += w * a.y; sa.z += w * a.z; sa.w += w * a.w;
        sb.x += w * b.x; sb.y += w * b.y; sb.z += w * b.z; sb.w += w * b.w;
      }
      const uint32_t entry = base + e;
      // (entries are owned by one CTA, whose chunks are ordered by __syncthreads: the stamp read sees its earlier chunks)
      const bool fresh = stamped && stamp[entry] != mark;
      if (stamped) stamp[entry] = mark;
      float4* dst = reinterpret_cast<float4*>(gtable + (size_t)entry * FIT_F);
      const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
      float4 x = fresh ? z4 : dst[0], y = fresh ? z4 : dst[1];
      x.x += sa.x; x.y += sa.y; x.z += sa.z; x.w += sa.w;
      y.x += sb.x; y.y += sb.y; y.z += sb.z; y.w += sb.w;
      dst[0] = x;
      dst[1] = y;
    }
    __syncthreads();  // the next chunk reuses the keys and the counter
  }
}

// gather bank rows (fp32) -> hi/lo planes [n, ld] (input of the residual MLP)
__global__ void fit_gather_rows_kernel(const float* __restrict__ bank, int C, StepRows sr, int n,
                                       float* __restrict__ out, int ld, size_t plane) {
  pdl_wait();     // (no-ops unless launched with programmatic stream serialisation)
  pdl_trigger();
  const int i = blockIdx.x;
  const int* rows = sr.rows(n);
  const float4* src = reinterpret_cast<const float4*>(sr.bank(bank) + (size_t)(rows ? rows[i] : i) * C);
  for (int c4 = threadIdx.x; c4 < C / 4; c4 += blockDim.x) {
    const float4 v = __ldg(src + c4);
    const float4 hi = make_float4(tf32_hi(v.x), tf32_hi(v.y), tf32_hi(v.z), tf32_hi(v.w));
    float* dst = out + (size_t)i * ld + c4 * 4;
    *reinterpret_cast<float4*>(dst) = hi;
    *reinterpret_cast<float4*>(dst + plane) = make_float4(v.x - hi.x, v.y - hi.y, v.z - hi.z, v.w - hi.w);
  }
}

// ----------------------------------------------------------------------------------------------------
// loss + gradient kernel: one warp per sampled row (C % 4 == 0, C <= 1536).
// losses[5] (this step's slots) accumulates: total, patch_l2, cosine, residual, residual_sparsity.
// ----------------------------------------------------------------------------------------------------
struct LossArgs {
  const float* raw;         // [2 planes][n, ld_raw] raw ViT features of the sampled rows (hi / lo, gathered on a side stream:
                            //  random 3 KB rows of a 3 GB bank are TLB misses that must not sit on the critical path)
  int ld_raw;
  size_t raw_plane;
  StepRows sr;              // bank rows of this step
  const float* F;           // [n, C] field output
  const float* G;           // [hw, C] shared artifact map (fp32 master)
  const float* R;           // [n, C] residual prediction or nullptr (phase 1)
  float* dpred;             // [2 planes][n, C] (hi / lo)
  float* dR;                // [2 planes][n, C] or nullptr
  size_t plane;             // n * C
  float* gG;                // [hw, C] gradient accumulator or nullptr (G frozen)
  float* losses;            // [num_iters, 5]; this step's slots are used
  int n, C, hw;
  float loss_scale;
  // F.grid_sample(G, coords, bilinear, align_corners=True) at the reference's linspace(-1, 1) node coordinates: in fp32
  // a node's unnormalised position ((x + 1) / 2) * (size - 1) is not always the integer it stands for, so the sample
  // reads (and its gradient reaches) a neighbouring cell with a weight of ~1e-6.  Adam normalises gradients, so that
  // leakage decides the update of cells that were not sampled themselves.  Per axis node: first cell, weight of that cell,
  // weight of the next one (oracle/fit.py::artifact_axis_table; nullptr: plain cell indexing).
  const int* ax_i0;         // [gw] x nodes then [gh] y nodes
  const float* ax_w0;
  const float* ax_w1;
  int gw, gh;
};

// NV = float4 per lane (ceil(C / 128)); all global loads of a row are issued before the first use.
template <int NV, bool HAS_R>
__global__ void __launch_bounds__(256, 2) fit_loss_kernel(LossArgs a) {
  pdl_wait();     // (no-ops unless launched with programmatic stream serialisation)
  pdl_trigger();
  const int row_raw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const bool row_ok = row_raw < a.n;       // (whole warps; the CTA still meets at the __syncthreads below)
  const int row = row_ok ? row_raw : a.n - 1;
  const int C = a.C, nvec = row_ok ? (a.C >> 2) : 0;  // a warp without a row loads / stores nothing
  const int br = a.sr.rows(a.n)[row];
  float* losses = a.losses + (size_t)a.sr.step() * 5;
  const int cell = br % a.hw;  // (r, c) of the patch inside its view: the "shared artifact coordinate"
  // the cell grid_sample reads for this node and its bilinear weight: per axis the heavier of the two corners (always
  // inside the map).  The ~1e-6 share of the lighter corners is below one ulp of pred and is not read here; their share of
  // the GRADIENT is what Adam amplifies, and fit_g_scatter_kernel delivers it.
  int cmain = cell;
  float wmain = 1.f;
  if (a.ax_i0) {
    const int cy = cell / a.gw, cx = cell - cy * a.gw;
    const bool nx = a.ax_w1[cx] > a.ax_w0[cx], ny = a.ax_w1[a.gw + cy] > a.ax_w0[a.gw + cy];
    cmain = (a.ax_i0[a.gw + cy] + (ny ? 1 : 0)) * a.gw + a.ax_i0[cx] + (nx ? 1 : 0);
    wmain = (nx ? a.ax_w1[cx] : a.ax_w0[cx]) * (ny ? a.ax_w1[a.gw + cy] : a.ax_w0[a.gw + cy]);
  }
  const float4* raw4 = reinterpret_cast<const float4*>(a.raw + (size_t)row * a.ld_raw);
  const float4* raw4lo = reinterpret_cast<const float4*>(a.raw + a.raw_plane + (size_t)row * a.ld_raw);
  const float4* F4 = reinterpret_cast<const float4*>(a.F + (size_t)row * C);
  const float4* R4 = HAS_R ? reinterpret_cast<const float4*>(a.R + (size_t)row * C) : nullptr;
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 pred[NV], raw[NV], rp[HAS_R ? NV : 1];
  {
    float4 f[NV], gg[NV], rl[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) {  // loads only
      const int v = lane + 32 * i;
      const bool ok = v < nvec;
      f[i] = ok ? F4[v] : z4;
      {  // the sampled value: the node's own cell times its corner weight.  (The ~1e-6 share of a neighbouring cell that
         // grid_sample adds for 9 of 37 nodes changes pred by less than one fp32 ulp; reading it cost 5-10 us per step on
         // the critical path.  The GRADIENT share of the neighbours is what Adam amplifies: fit_g_scatter_kernel keeps it.)
        const float4 t = ok ? __ldg(reinterpret_cast<const float4*>(a.G + (size_t)cmain * C) + v) : z4;
        gg[i] = make_float4(t.x * wmain, t.y * wmain, t.z * wmain, t.w * wmain);
      }
      raw[i] = ok ? raw4[v] : z4;
      rl[i] = ok ? raw4lo[v] : z4;
      if (HAS_R) rp[i] = ok ? R4[v] : z4;
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      raw[i] = make_float4(raw[i].x + rl[i].x, raw[i].y + rl[i].y, raw[i].z + rl[i].z, raw[i].w + rl[i].w);  // hi + lo == raw
      pred[i] = make_float4(f[i].x + gg[i].x, f[i].y + gg[i].y, f[i].z + gg[i].z, f[i].w + gg[i].w);
      if (HAS_R) { pred[i].x += rp[i].x; pred[i].y += rp[i].y; pred[i].z += rp[i].z; pred[i].w += rp[i].w; }
    }
  }
  float dot = 0.f, pp = 0.f, rr = 0.f, sse = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {  // lanes beyond nvec hold zeros: they add nothing
    const float4 p = pred[i], r = raw[i];
    dot += p.x * r.x + p.y * r.y + p.z * r.z + p.w * r.w;
    pp += p.x * p.x + p.y * p.y + p.z * p.z + p.w * p.w;
    rr += r.x * r.x + r.y * r.y + r.z * r.z + r.w * r.w;
    const float dx = p.x - r.x, dy = p.y - r.y, dz = p.z - r.z, dw = p.w - r.w;
    sse += dx * dx + dy * dy + dz * dz + dw * dw;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {  // four reductions interleaved
    dot += __shfl_xor_sync(0xffffffffu, dot, o);
    pp += __shfl_xor_sync(0xffffffffu, pp, o);
    rr += __shfl_xor_sync(0xffffffffu, rr, o);
    sse += __shfl_xor_sync(0xffffffffu, sse, o);
  }
  const float np_ = fmaxf(sqrtf(pp), 1e-8f), nr_ = fmaxf(sqrtf(rr), 1e-8f);  // F.cosine_similarity eps
  const float cosv = dot / (np_ * nr_);
  const float inv_nc = 1.f / ((float)a.n * (float)C), inv_n = 1.f / (float)a.n;
  // d/dpred [ mean((p-r)^2) + 1 - mean_rows cos ] * loss_scale
  const float k_mse = 2.f * inv_nc * a.loss_scale;
  const float k_cr = -inv_n * a.loss_scale / (np_ * nr_);        // coefficient of raw
  const float k_cp = inv_n * a.loss_scale * cosv / (np_ * np_);  // coefficient of pred
  float res_sq = 0.f, res_abs = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int v = lane + 32 * i;
    if (v >= nvec) continue;
    const float4 p = pred[i], r = raw[i];
    float4 d;
    d.x = k_mse * (p.x - r.x) + k_cr * r.x + k_cp * p.x;
    d.y = k_mse * (p.y - r.y) + k_cr * r.y + k_cp * p.y;
    d.z = k_mse * (p.z - r.z) + k_cr * r.z + k_cp * p.z;
    d.w = k_mse * (p.w - r.w) + k_cr * r.w + k_cp * p.w;
    {
      const float4 hi = make_float4(tf32_hi(d.x), tf32_hi(d.y), tf32_hi(d.z), tf32_hi(d.w));
      float* dp = a.dpred + (size_t)row * C + v * 4;
      *reinterpret_cast<float4*>(dp) = hi;
      *reinterpret_cast<float4*>(dp + a.plane) = make_float4(d.x - hi.x, d.y - hi.y, d.z - hi.z, d.w - hi.w);
    }
    if (HAS_R) {
      // gt_residual = raw - denoised - shared = raw - (pred - R); e = R - gt = pred - raw
      const float4 q = rp[i];
      const float ex = p.x - r.x, ey = p.y - r.y, ez = p.z - r.z, ew = p.w - r.w;
      res_sq += ex * ex + ey * ey + ez * ez + ew * ew;
      res_abs += fabsf(q.x) + fabsf(q.y) + fabsf(q.z) + fabsf(q.w);
      const float k1 = 0.2f * inv_nc * a.loss_scale, k2 = 0.02f * inv_nc * a.loss_scale;
      auto sgn = [](float x) { return (float)((x > 0.f) - (x < 0.f)); };
      const float4 dr = make_float4(k1 * ex + k2 * sgn(q.x), k1 * ey + k2 * sgn(q.y), k1 * ez + k2 * sgn(q.z),
                                    k1 * ew + k2 * sgn(q.w));
      const float4 hi = make_float4(tf32_hi(dr.x), tf32_hi(dr.y), tf32_hi(dr.z), tf32_hi(dr.w));
      float* dp = a.dR + (size_t)row * C + v * 4;
      *reinterpret_cast<float4*>(dp) = hi;
      *reinterpret_cast<float4*>(dp + a.plane) = make_float4(dr.x - hi.x, dr.y - hi.y, dr.z - hi.z, dr.w - hi.w);
    }
  }
  if (HAS_R) {
    res_sq = warp_sum(res_sq);
    res_abs = warp_sum(res_abs);
  }
  // loss logging: reduce over the 8 warps of the CTA first -- 2048 warps x 5 atomics on ONE cache line serialise in L2
  // and used to cost ~20 us of the 25 us this kernel took.
  __shared__ float s_part[8][5];
  const int wib = threadIdx.x >> 5;
  if (lane == 0) {
    const float l2 = sse * inv_nc, lc = (1.f - cosv) * inv_n;
    const float lr = 0.1f * res_sq * inv_nc, ls = 0.02f * res_abs * inv_nc;
    s_part[wib][0] = l2 + lc + lr + ls;
    s_part[wib][1] = l2;
    s_part[wib][2] = lc;
    s_part[wib][3] = lr;
    s_part[wib][4] = ls;
  }
  __syncthreads();
  if (threadIdx.x < 5 && (HAS_R || threadIdx.x < 3)) {
    float t = 0.f;
    const int nw = min(8, a.n - (int)(blockIdx.x * (blockDim.x >> 5)));  // warps of this CTA that own a row
#pragma unroll
    for (int k = 0; k < 8; ++k)
      if (k < nw) t += s_part[k][threadIdx.x];
    atomicAdd(losses + threadIdx.x, t);
  }
}

// dG of phase 1, off the critical path: the loss kernel stores d pred (hi / lo planes); this kernel, on a side stream,
// adds every row's d pred to the cells of G that F.grid_sample reads for the row's node (normally one cell with weight 1,
// for 9 of 37 nodes per axis also a neighbour with a weight of ~1e-6: see LossArgs).  Only Adam(small) at the end of the
// step consumes gG, so nothing on the main stream waits for it.  One warp per cell GATHERS the rows that touch it, in
// ascending row order: the sum does not depend on thread scheduling (with atomics it would, and Adam amplifies that).
struct ScatterArgs {
  const float* dpred;       // [2 planes][n, C]
  size_t plane;
  StepRows sr;
  float* gG;                // [hw, C]
  int n, C, hw, gw, gh;
  const int* ax_i0;
  const float* ax_w0;
  const float* ax_w1;
};
constexpr int GS_MAXV = 1536 / 4 / 32;  // float4 columns per lane (C <= 1536)
__global__ void __launch_bounds__(256) fit_g_scatter_kernel(ScatterArgs a) {
  pdl_wait();
  pdl_trigger();
  const int cell = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (cell >= a.hw) return;
  const int* rows = a.sr.rows(a.n);
  const int ty = cell / a.gw, tx = cell - ty * a.gw;
  const int nv = a.C >> 2;
  float4 acc[GS_MAXV];
#pragma unroll
  for (int j = 0; j < GS_MAXV; ++j) acc[j] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int r0 = 0; r0 < a.n; r0 += 32) {
    // weight with which row r0 + lane reaches this cell (0: it does not)
    float w = 0.f;
    const int row = r0 + lane;
    if (row < a.n) {
      const int rc = rows[row] % a.hw;
      if (!a.ax_i0) {
        w = rc == cell ? 1.f : 0.f;
      } else {
        const int cy = rc / a.gw, cx = rc - cy * a.gw;
        const int x0 = a.ax_i0[cx], y0 = a.ax_i0[a.gw + cy];
        const int dx = tx - x0, dy = ty - y0;
        if (dx >= 0 && dx <= 1 && dy >= 0 && dy <= 1)
          w = (dx ? a.ax_w1[cx] : a.ax_w0[cx]) * (dy ? a.ax_w1[a.gw + cy] : a.ax_w0[a.gw + cy]);
      }
    }
    unsigned hit = __ballot_sync(0xffffffffu, w != 0.f);
    while (hit) {
      const int src = __ffs(hit) - 1;
      hit &= hit - 1;
      const float wk = __shfl_sync(0xffffffffu, w, src);
      const float4* hi = reinterpret_cast<const float4*>(a.dpred + (size_t)(r0 + src) * a.C);
      const float4* lo = reinterpret_cast<const float4*>(a.dpred + a.plane + (size_t)(r0 + src) * a.C);
#pragma unroll
      for (int j = 0; j < GS_MAXV; ++j) {
        const int v = lane + 32 * j;
        if (v < nv) {
          const float4 h = hi[v], l = lo[v];
          const float4 d = make_float4(h.x + l.x, h.y + l.y, h.z + l.z, h.w + l.w);  // hi + lo == d pred exactly
          acc[j].x += d.x * wk; acc[j].y += d.y * wk; acc[j].z += d.z * wk; acc[j].w += d.w * wk;
        }
      }
    }
  }
  float4* dst = reinterpret_cast<float4*>(a.gG + (size_t)cell * a.C);
#pragma unroll
  for (int j = 0; j < GS_MAXV; ++j) {
    const int v = lane + 32 * j;
    if (v < nv) {
      float4 x = dst[v];
      x.x += acc[j].x; x.y += acc[j].y; x.z += acc[j].z; x.w += acc[j].w;
      dst[v] = x;
    }
  }
}

template <bool HAS_R>
static int launch_loss_nv(const LossArgs& la, int blocks, int tb, cudaStream_t st, bool pdl) {
  const int nv = (la.C / 4 + 31) / 32;
  const dim3 g(blocks), b(tb);
  if (nv <= 1) DVT_CUDA_OK(launch_k(pdl, fit_loss_kernel<1, HAS_R>, g, b, 0, st, la));
  else if (nv <= 2) DVT_CUDA_OK(launch_k(pdl, fit_loss_kernel<2, HAS_R>, g, b, 0, st, la));
  else if (nv <= 3) DVT_CUDA_OK(launch_k(pdl, fit_loss_kernel<3, HAS_R>, g, b, 0, st, la));
  else if (nv <= 6) DVT_CUDA_OK(launch_k(pdl, fit_loss_kernel<6, HAS_R>, g, b, 0, st, la));
  else if (nv <= 8) DVT_CUDA_OK(launch_k(pdl, fit_loss_kernel<8, HAS_R>, g, b, 0, st, la));
  else DVT_CUDA_OK(launch_k(pdl, fit_loss_kernel<12, HAS_R>, g, b, 0, st, la));
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

static int launch_loss(const LossArgs& la, cudaStream_t st, bool pdl) {
  const int tb = 256, blocks = (la.n * 32 + tb - 1) / tb;
  return la.R ? launch_loss_nv<true>(la, blocks, tb, st, pdl) : launch_loss_nv<false>(la, blocks, tb, st, pdl);
}

// ----------------------------------------------------------------------------------------------------
// Adam (torch.optim.Adam semantics: L2 weight decay folded into the gradient, bias-corrected, eps outside sqrt)
//   g' = g + wd p;  m += (g' - m)(1-b1);  v = b2 v + (1-b2) g'^2;  p -= step_size * m / (sqrt(v)/bc2_sqrt + eps)
// step_size = lr/(1-b1^t) and bc2_sqrt = sqrt(1-b2^t) are precomputed per step in double on the host.
// ----------------------------------------------------------------------------------------------------
// (AdamScalars / adam1() are defined above, next to the encode kernel that also applies them.)

// Dense sweep of the window of steps [b, b + len), len <= KW: S_{b+len} = Adam^len(S_b, g_b .. g_{b+len-1}), read
// from state buffer (step_base[1] + buf_off) & 1, written to the other one.  Every element is loaded once, takes the
// len Adam steps in registers, one after another (the same adam1() on the same inputs as len one-step sweeps, so the
// stored bits are the same), and is stored once: 24 B/param per window + len stamp reads per entry.  Gradients are
// read for stamped entries only.
// Launch geometries (fit_sweep_geometry): many short-lived 256-thread CTAs (fastest alone: 77 us, the HBM peak), or a
// few persistent 1024-thread CTAs that fill one SM each and leave the other SMs to the GEMM chain of the next steps.
// (Measured and rejected: one contiguous slice per CTA -- 133 us, HBM channel imbalance; maximum shared-memory
// carve-out -- 137 us.)
template <int KW>
__global__ void __launch_bounds__(1024, 1)
fit_adam_table_kernel(TableBufs tb, size_t nvec, const AdamScalars* __restrict__ sc, const int* __restrict__ step_base,
                      int step_off, int len, int buf_off, float wd) {
  // two elements in flight per thread for one-step windows, one for longer windows; the gradient loads of windows over 4
  // steps wait for their Adam step instead of being issued with p, m, v (registers: 64 per thread at 1024 threads)
  constexpr int ADAM_UNROLL = KW == 1 ? 2 : 1;
  constexpr bool HOIST = KW <= 4;
  pdl_wait();     // (no-ops unless launched with programmatic stream serialisation)
  pdl_trigger();
  const int b = step_base[0] + step_off;
  const int src = (step_base[1] + buf_off) & 1;
  const float4* __restrict__ p = reinterpret_cast<const float4*>(DVT_SEL2(tb.p, src));
  const float4* __restrict__ m = reinterpret_cast<const float4*>(DVT_SEL2(tb.m, src));
  const float4* __restrict__ v = reinterpret_cast<const float4*>(DVT_SEL2(tb.v, src));
  float4* __restrict__ po = reinterpret_cast<float4*>(DVT_SEL2(tb.p, src ^ 1));
  float4* __restrict__ mo = reinterpret_cast<float4*>(DVT_SEL2(tb.m, src ^ 1));
  float4* __restrict__ vo = reinterpret_cast<float4*>(DVT_SEL2(tb.v, src ^ 1));
  // grid-stride: all CTAs advance one contiguous front together, which spreads the traffic evenly over the HBM channels
  const size_t hi = nvec;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  // ring slot of step b + j: slot(b) + j, wrapped (len <= KW <= ring / 2)
  auto slot_ofs = [&](int j) -> size_t {
    int s = tb.slot(b) + j;
    s -= s >= tb.ring ? tb.ring : 0;
    return (size_t)s * tb.n_entries;
  };
  // The gradient loads depend on the stamps; stamps are therefore fetched one iteration ahead so that the (rare)
  // gradient loads are issued together with p, m, v instead of one DRAM latency later.
  uint32_t st_next[ADAM_UNROLL][KW];
  {
    const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
#pragma unroll
    for (int u = 0; u < ADAM_UNROLL; ++u) {
      const size_t i = i0 + u * stride;
#pragma unroll
      for (int j = 0; j < KW; ++j)
        st_next[u][j] = (j < len && i < hi) ? __ldg(tb.stamp + slot_ofs(j) + (i >> 1)) : 0u;
    }
  }
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < hi; i0 += ADAM_UNROLL * stride) {
    float4 pp[ADAM_UNROLL], mm[ADAM_UNROLL], vv[ADAM_UNROLL], gg[ADAM_UNROLL][HOIST ? KW : 1];
    uint32_t st[ADAM_UNROLL][HOIST ? 1 : KW];
    bool ok[ADAM_UNROLL];
#pragma unroll
    for (int u = 0; u < ADAM_UNROLL; ++u) {
      const size_t i = i0 + u * stride;
      ok[u] = i < hi;
      if (ok[u]) { pp[u] = p[i]; mm[u] = m[i]; vv[u] = v[i]; }
      const size_t inext = i + ADAM_UNROLL * stride;
#pragma unroll
      for (int j = 0; j < KW; ++j) {
        if constexpr (HOIST) {
          gg[u][j] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok[u] && j < len && st_next[u][j] == (uint32_t)(b + j) + 1u)  // entry = 8 floats = 2 float4
            gg[u][j] = reinterpret_cast<const float4*>(tb.g + slot_ofs(j) * FIT_F)[i];
        } else {
          st[u][j] = st_next[u][j];
        }
        st_next[u][j] = (j < len && inext < hi) ? __ldg(tb.stamp + slot_ofs(j) + (inext >> 1)) : 0u;
      }
    }
#pragma unroll
    for (int u = 0; u < ADAM_UNROLL; ++u) {
      if (!ok[u]) continue;
      const size_t i = i0 + u * stride;
#pragma unroll
      for (int j = 0; j < KW; ++j) {
        if (j >= len) break;
        float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (HOIST) g = gg[u][j];
        else if (st[u][j] == (uint32_t)(b + j) + 1u) g = reinterpret_cast<const float4*>(tb.g + slot_ofs(j) * FIT_F)[i];
        const AdamScalars s = sc[b + j];
        adam1(pp[u].x, mm[u].x, vv[u].x, g.x, wd, s.step_size, s.inv_bc2_sqrt);
        adam1(pp[u].y, mm[u].y, vv[u].y, g.y, wd, s.step_size, s.inv_bc2_sqrt);
        adam1(pp[u].z, mm[u].z, vv[u].z, g.z, wd, s.step_size, s.inv_bc2_sqrt);
        adam1(pp[u].w, mm[u].w, vv[u].w, g.w, wd, s.step_size, s.inv_bc2_sqrt);
      }
      po[i] = pp[u]; mo[i] = mm[u]; vo[i] = vv[u];
    }
  }
}

// ----------------------------------------------------------------------------------------------------
// EXPERIMENT (DVT_FIT_SWEEP_TMA=1; not the default): the same sweep staged through shared memory by bulk async copies
// (TMA, cp.async.bulk).  One-step windows only (the host runs the plain kernel for longer ones).  ONE thread per CTA
// keeps three 50 KB chunks (p, m, v and the stamps of 512 table entries) in flight per SM through an mbarrier ring of four stages while 512 threads run the Adam arithmetic out of
// shared memory and write the results back with coalesced 16-byte stores.  Idea: memory-level parallelism independent of
// the thread count, so that a few dozen SMs could saturate HBM (Little's law: the bytes in flight per SM times the SMs
// the sweep runs on, over the loaded latency, bound its rate).  Same adam1() arithmetic, same stamp rules:
// bit-identical results (tests/test_fit_gpu.py::test_sweep_kernels_agree).
// Chunks are dealt round-robin (chunk c -> CTA c % grid), i.e. all CTAs advance one contiguous front together.
// ----------------------------------------------------------------------------------------------------
constexpr int SW_ENT = 512;                       // table entries per chunk
constexpr int SW_FLOATS = SW_ENT * FIT_F;         // 4096 floats = 16 KB per array and chunk
constexpr int SW_STAGES = 4;
constexpr int SW_THREADS = 512;
struct SweepStage {
  float p[SW_FLOATS], m[SW_FLOATS], v[SW_FLOATS];
  uint32_t stamp[SW_ENT];
};
constexpr size_t SW_SMEM = SW_STAGES * sizeof(SweepStage) + SW_STAGES * sizeof(uint64_t) + 128;
static_assert(sizeof(SweepStage) % 128 == 0, "stage size keeps the 16-byte alignment of bulk copies");
static_assert(SW_SMEM <= 227 * 1024, "sweep stages exceed shared memory");

__global__ void __launch_bounds__(SW_THREADS, 1)
fit_adam_table_tma_kernel(TableBufs tb, uint32_t n_entries, const AdamScalars* __restrict__ sc,
                          const int* __restrict__ step_base, int step_off, int buf_off, float wd) {
  extern __shared__ uint8_t sw_smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sw_smem_raw) + 127) & ~uintptr_t(127));
  SweepStage* stg = reinterpret_cast<SweepStage*>(base);
  uint64_t* full = reinterpret_cast<uint64_t*>(base + SW_STAGES * sizeof(SweepStage));
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < SW_STAGES; ++s) mbar_init(&full[s], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();     // (no-ops unless launched with programmatic stream serialisation)
  pdl_trigger();
  const int step = step_base[0] + step_off;
  const int src = (step_base[1] + buf_off) & 1;
  const float* __restrict__ p = DVT_SEL2(tb.p, src);
  const float* __restrict__ m = DVT_SEL2(tb.m, src);
  const float* __restrict__ v = DVT_SEL2(tb.v, src);
  float4* __restrict__ po = reinterpret_cast<float4*>(DVT_SEL2(tb.p, src ^ 1));
  float4* __restrict__ mo = reinterpret_cast<float4*>(DVT_SEL2(tb.m, src ^ 1));
  float4* __restrict__ vo = reinterpret_cast<float4*>(DVT_SEL2(tb.v, src ^ 1));
  const float4* __restrict__ g = reinterpret_cast<const float4*>(tb.g_of(step));
  const uint32_t* __restrict__ stamp = tb.stamp_of(step);
  const AdamScalars s = sc[step];
  const uint32_t mark = (uint32_t)step + 1u;
  const uint32_t n_chunks = (n_entries + SW_ENT - 1) / SW_ENT;

  auto issue = [&](uint32_t k) {  // thread 0: bulk loads of this CTA's k-th chunk into stage k % SW_STAGES
    const uint32_t c = blockIdx.x + k * gridDim.x;
    if (c >= n_chunks) return;
    SweepStage& st = stg[k % SW_STAGES];
    uint64_t* bar = &full[k % SW_STAGES];
    const uint32_t e0 = c * SW_ENT, ne = min((uint32_t)SW_ENT, n_entries - e0);
    const uint32_t bp = ne * FIT_F * 4, bs = ne * 4;  // entries per level are multiples of 8: both multiples of 32 B
    mbar_expect_tx(bar, 3 * bp + bs);
    bulk_load_1d(st.p, p + (size_t)e0 * FIT_F, bp, bar);
    bulk_load_1d(st.m, m + (size_t)e0 * FIT_F, bp, bar);
    bulk_load_1d(st.v, v + (size_t)e0 * FIT_F, bp, bar);
    bulk_load_1d(st.stamp, stamp + e0, bs, bar);
  };
  if (tid == 0)
    for (uint32_t k = 0; k + 1 < SW_STAGES; ++k) issue(k);

  for (uint32_t k = 0;; ++k) {
    const uint32_t c = blockIdx.x + k * gridDim.x;
    if (c >= n_chunks) break;
    // refill the stage that was consumed in iteration k-1 (all its readers passed the __syncthreads below)
    if (tid == 0) issue(k + SW_STAGES - 1);
    const SweepStage& st = stg[k % SW_STAGES];
    mbar_wait(&full[k % SW_STAGES], (k / SW_STAGES) & 1u, 0x51);
    const uint32_t e0 = c * SW_ENT, ne = min((uint32_t)SW_ENT, n_entries - e0);
    const size_t f0 = (size_t)e0 * 2;            // first float4 of the chunk
    const float4* sp = reinterpret_cast<const float4*>(st.p);
    const float4* sm = reinterpret_cast<const float4*>(st.m);
    const float4* sv = reinterpret_cast<const float4*>(st.v);
#pragma unroll
    for (int u = 0; u < (SW_ENT * 2) / SW_THREADS; ++u) {
      const uint32_t i = tid + u * SW_THREADS;   // float4 index inside the chunk; entry = i / 2
      if (i < ne * 2) {
        const bool touched = st.stamp[i >> 1] == mark;
        float4 pp = sp[i], mm = sm[i], vv = sv[i];
        float4 gg = make_float4(0.f, 0.f, 0.f, 0.f);
        if (touched) gg = __ldcg(g + f0 + i);
        adam1(pp.x, mm.x, vv.x, gg.x, wd, s.step_size, s.inv_bc2_sqrt);
        adam1(pp.y, mm.y, vv.y, gg.y, wd, s.step_size, s.inv_bc2_sqrt);
        adam1(pp.z, mm.z, vv.z, gg.z, wd, s.step_size, s.inv_bc2_sqrt);
        adam1(pp.w, mm.w, vv.w, gg.w, wd, s.step_size, s.inv_bc2_sqrt);
        po[f0 + i] = pp; mo[f0 + i] = mm; vo[f0 + i] = vv;
      }
    }
    __syncthreads();
  }
}

// small params: one flat buffer; [g_lo, g_hi) is G, [r_lo, r_hi) the residual MLP, the rest the field MLP.
__global__ void fit_adam_small_kernel(float4* __restrict__ p, float4* __restrict__ m, float4* __restrict__ v,
                                      float4* __restrict__ g, float* __restrict__ wsplit, int nvec, int g_lo,
                                      int g_hi, int r_lo, int r_hi, const AdamScalars* __restrict__ sc_main,
                                      const AdamScalars* __restrict__ sc_res, const int* __restrict__ step_base,
                                      int step_off, int freeze_step, float wd) {
  pdl_wait();     // (no-ops unless launched with programmatic stream serialisation)
  pdl_trigger();
  const int step = *step_base + step_off;
  const bool phase2 = step > freeze_step;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += gridDim.x * blockDim.x) {
    const bool is_g = i >= g_lo && i < g_hi, is_r = i >= r_lo && i < r_hi;
    if ((is_g && phase2) || (is_r && !phase2)) continue;  // grad is None in the reference: Adam skips the tensor
    const AdamScalars s = is_r ? sc_res[step] : sc_main[step];
    float4 pp = p[i], mm = m[i], vv = v[i];
    const float4 gg = g[i];
    adam1(pp.x, mm.x, vv.x, gg.x, wd, s.step_size, s.inv_bc2_sqrt);
    adam1(pp.y, mm.y, vv.y, gg.y, wd, s.step_size, s.inv_bc2_sqrt);
    adam1(pp.z, mm.z, vv.z, gg.z, wd, s.step_size, s.inv_bc2_sqrt);
    adam1(pp.w, mm.w, vv.w, gg.w, wd, s.step_size, s.inv_bc2_sqrt);
    p[i] = pp; m[i] = mm; v[i] = vv;
    g[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!is_g) {  // GEMM operand planes of the weights
      const float4 hi = make_float4(tf32_hi(pp.x), tf32_hi(pp.y), tf32_hi(pp.z), tf32_hi(pp.w));
      *reinterpret_cast<float4*>(wsplit + (size_t)i * 4) = hi;
      *reinterpret_cast<float4*>(wsplit + (size_t)(nvec + i) * 4) =
          make_float4(pp.x - hi.x, pp.y - hi.y, pp.z - hi.z, pp.w - hi.w);
    }
  }
}

// step_base[0]: step counter; step_base[1]: table sweeps since fit_begin (parity = state buffer of the current step)
__global__ void fit_advance_kernel(int* step_base, int steps, int sweeps) {
  step_base[0] += steps;
  step_base[1] += sweeps;
}

__global__ void fit_fill_col_kernel(float* buf, int ld, int col, int rows, float val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < rows) buf[(size_t)i * ld + col] = val;
}

__global__ void fit_transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int rows, int cols) {
  // out[c, r] = in[r, c]
  const size_t total = (size_t)rows * cols;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
    const size_t r = e / cols, c = e - r * cols;
    out[c * rows + r] = in[e];
  }
}

// TF32 hi / lo operand planes of n parameters: wsplit[e] = hi, wsplit[plane + e] = lo
__global__ void fit_split_kernel(const float* __restrict__ p, float* __restrict__ wsplit, size_t n, size_t plane) {
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    const float v = p[e], hi = tf32_hi(v);
    wsplit[e] = hi;
    wsplit[plane + e] = v - hi;
  }
}

__global__ void fit_coord_range_kernel(const float* __restrict__ coords, size_t n2, int* __restrict__ bad) {
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n2; e += (size_t)gridDim.x * blockDim.x) {
    const float c = coords[e];
    if (!(c >= 0.f && c <= 1.f)) atomicExch(bad, 1);
  }
}

// ====================================================================================================
// host engine
// ====================================================================================================
#define FIT_RC0(x) do { int _rc0 = (x); if (_rc0) return _rc0; } while (0)
struct Seg {
  int off = 0, rows = 0, cols = 0;  // floats; weights are [rows, cols] row-major, biases rows x 1
};

constexpr int FIT_SEM_TILES = 1024;

struct Fit {
  // config
  int C, gh, gw, hw, bsz, Lf;
  GridLevels grid;
  size_t n_table;  // floats
  // small-param layout (offsets in floats, multiples of 8)
  Seg W1, b1, W2, b2, G, R1, rb1, R2, rb2, R3, rb3;
  int n_small = 0;
  // device memory
  TableBufs tb = {};                           // ping-pong p/m/v, ring of gradient / stamp slots
  int cur_host = 0;                            // steps completed (host view)
  int cur_buf = 0;                             // table sweeps completed mod 2 (host view): the current table is tb.p[cur_buf]
  cudaStream_t sD = nullptr;                   // stream of the pipelined table sweeps
  cudaEvent_t ev_sweep[3] = {};                // completion of the window sweep w of the epoch (slot w % 3)
  // Epoch = the steps enqueued since the sweeps were last joined (a graph, or one plain step); its windows are counted from 0
  int epoch_steps = 0;                         // steps enqueued in this epoch
  int epoch_windows = 0;                       // table sweeps enqueued in this epoch (the open window's index)
  int win_first = 0, prev_first = 0;           // epoch step of the first step of the open window / of the window before
  bool epoch_forked = false;                   // this epoch forked sweeps onto sD (pipelined schedule)
  int sweep_steps[2] = {4, 4};                 // DVT_FIT_SWEEP_STEPS "k1,k2": window of the pipelined sweep per phase
  bool enc_ready = false;                      // f->enc already holds the encoding of the next step
  int res_x3 = 1;                              // GEMM mode of the residual MLP: 1 = 3xTF32, 2 = plain TF32 (experiment)
  int sweep_threads = 1024;                    // DVT_FIT_SWEEP_THREADS: threads of a persistent sweep CTA (1024 fills the register file of
                                               // its SM; 512 leaves half of it to co-resident CTAs of the chain)
  int x3_wide_min_n[2] = {0, 256};             // DVT_FIT_X3_WIDE_MIN_N "p1,p2": 128 x 128 GEMM tiles when N >= this (0: never)
  int wgrad_sms = 96;                          // DVT_FIT_WGRAD_SMS: weight-gradient GEMMs split K to fill at most this many SMs
  bool sweep_pdl = true;                       // DVT_FIT_SWEEP_PDL=0: the persistent sweep CTAs of step t+1 are not made resident
                                               // (waiting, one full SM each) while sweep t still runs
  int off_path_prio_drop = 0;                  // DVT_FIT_OFFPATH_PRIO: priority levels below the chain for off-path kernels
  int wgrad_x3 = 1;                            // GEMM mode of the field MLP's weight-gradient GEMMs (DVT_FIT_WGRAD_TF32=1: 2)
  bool pdl = true;                             // programmatic dependent launch along the kernel chains of a step
  bool pipe[2] = {true, true};                 // software-pipelined table sweep in phase 1 / 2 (see fit_enqueue_step)
  int sweep_ctas[2] = {0, 0};                  // persistent sweep CTAs in phase 1 / 2 (0 = many small CTAs)
  bool sweep_tma = false;                      // DVT_FIT_SWEEP_TMA=1: persistent sweep = the TMA-staged kernel (experiment)
  float *sp = nullptr, *sm = nullptr, *sv = nullptr, *sg = nullptr;
  float* wsplit = nullptr;  // [2][n_small] TF32 hi / lo planes of the small params (x3 GEMM operands)
  // activations: GEMM operands are stored as two fp32 planes (hi, lo), plane stride = bsz * ld
  float *enc = nullptr, *h1 = nullptr, *dpred = nullptr, *dh1 = nullptr;
  float *Fout = nullptr, *denc = nullptr;
  float *rawb = nullptr, *r1 = nullptr, *r2 = nullptr, *dR = nullptr, *dr2 = nullptr, *dr1 = nullptr;
  float* Rout = nullptr;
  int ld_enc, ld_h1, ld_raw, ld_r;
  // schedule
  int num_iters = 0, freeze_step = 0;
  int cur_step = 0;                            // steps of the current schedule already enqueued (host mirror of *step_base)
  // sampling stream: two device buffers + two pinned staging buffers, so that the upload of the next image's stream
  // runs (on sU) while the current fit is still reading its own
  int* idx[2] = {nullptr, nullptr};            // [num_iters + 1, bsz] each
  int* idx_pinned[2] = {nullptr, nullptr};
  size_t idx_cap = 0;                          // elements per buffer
  int idx_slot = 1;                            // buffer of the current fit (toggled by fit_begin)
  cudaStream_t sU = nullptr;                   // upload stream
  cudaEvent_t ev_upload[2] = {};               // H2D of slot s complete
  cudaEvent_t ev_run_done[2] = {};             // last fit_run that read slot s complete
  bool run_done_valid[2] = {false, false};
  int* ax_i0 = nullptr;                        // grid_sample node tables of the artifact map (fit_set_artifact_grid), or null
  float *ax_w0 = nullptr, *ax_w1 = nullptr;
  int* flags_dev = nullptr;                    // bit 0: a coordinate outside [0, 1]; bit 1: a sampled row out of range
  int* flags_pinned = nullptr;
  double sched_key[6] = {-1, -1, -1, -1, -1, -1};  // (num_iters, warmup, lr, min_lr, freeze_step) of the uploaded tables
  AdamScalars *sc_main = nullptr, *sc_res = nullptr;
  float* losses = nullptr;    // [num_iters, 5]
  unsigned* wg_sem = nullptr; // [5][FIT_SEM_TILES] split-K counters of the five weight-gradient call sites (self-resetting)
  int* step_base = nullptr;
  float wd = 1e-5f, loss_scale = 1024.f;
  // bank (borrowed)
  const float* bank = nullptr;
  const float* coords = nullptr;
  size_t bank_rows = 0;
  FitInputs* inputs_dev = nullptr;  // device copy of {bank, coords}: what the (graph-captured) kernels dereference
  // graphs (captured on a stream owned by the engine: the caller's stream may be the legacy default stream,
  // which cannot be captured)
  cudaGraphExec_t graph1 = nullptr, graph2 = nullptr;
  int graph_steps = 0;
  long long graph1_nodes = 0, graph2_nodes = 0;
  int graph1_sweeps = 0, graph2_sweeps = 0;    // table sweeps per graph launch
  cudaStream_t stream = nullptr;      // main stream of a step (critical path)
  cudaStream_t sB = nullptr, sC = nullptr, sE = nullptr;  // side streams: independent GEMM chains beside the main one
  cudaEvent_t ev_in = nullptr, ev_out = nullptr;
  cudaEvent_t ev[16] = {};
  // query workspace
  int q_cap = 0;
  float *q_enc = nullptr, *q_h1 = nullptr, *q_raw = nullptr, *q_r1 = nullptr, *q_r2 = nullptr;
  float* q_stage = nullptr;
  size_t q_stage_cap = 0;
  std::vector<void*> owned;
};

// EXPERIMENT (DVT_FIT_CARVEOUT=<percent> for the small kernels, DVT_FIT_CARVEOUT_SWEEP=<percent> for the sweep; off by
// default).  The 3xTF32 GEMM CTAs of the chain need up to ~200 KB of shared memory, and an SM changes its L1 / shared-memory
// split only when it is idle: a GEMM CTA cannot join an SM on which one of the fit's small kernels (no shared memory, so by
// default the largest L1) got first.  Asking for a shared-memory carve-out on the fit's own kernels makes the GEMM CTAs
// resident beside them, at the cost of the L1 the sweep / encode / loss kernels keep their loads in flight in.
static int fit_prepare_kernels() {
  static bool done = false;
  if (done) return DVT_OK;
  done = true;
  DVT_CUDA_OK(cudaFuncSetAttribute(fit_grid_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GB_SMEM));
  const char* e = getenv("DVT_FIT_CARVEOUT");            // percent of the unified L1 / shared array, small kernels
  const char* es = getenv("DVT_FIT_CARVEOUT_SWEEP");     // ... the sweep
  const int pct = e ? atoi(e) : 0, pct_sweep = es ? atoi(es) : 0;
#define DVT_MAX_SHARED(k) DVT_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, pct))
  if (pct_sweep > 0) {
#define DVT_SWEEP_SHARED(k) DVT_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, pct_sweep))
    DVT_SWEEP_SHARED(fit_adam_table_kernel<1>); DVT_SWEEP_SHARED(fit_adam_table_kernel<2>);
    DVT_SWEEP_SHARED(fit_adam_table_kernel<4>); DVT_SWEEP_SHARED(fit_adam_table_kernel<8>);
#undef DVT_SWEEP_SHARED
  }
  if (pct <= 0) return DVT_OK;
  DVT_MAX_SHARED(fit_encode_kernel<2>); DVT_MAX_SHARED(fit_encode_kernel<4>); DVT_MAX_SHARED(fit_encode_kernel<8>);
  DVT_MAX_SHARED(fit_encode_kernel<10>); DVT_MAX_SHARED(fit_encode_kernel<16>);
  DVT_MAX_SHARED(fit_grid_bwd_kernel);
  DVT_MAX_SHARED(fit_gather_rows_kernel);
  DVT_MAX_SHARED(fit_g_scatter_kernel);
  DVT_MAX_SHARED(fit_adam_small_kernel);
  DVT_MAX_SHARED(fit_advance_kernel);
  DVT_MAX_SHARED((fit_loss_kernel<1, false>)); DVT_MAX_SHARED((fit_loss_kernel<1, true>));
  DVT_MAX_SHARED((fit_loss_kernel<2, false>)); DVT_MAX_SHARED((fit_loss_kernel<2, true>));
  DVT_MAX_SHARED((fit_loss_kernel<3, false>)); DVT_MAX_SHARED((fit_loss_kernel<3, true>));
  DVT_MAX_SHARED((fit_loss_kernel<6, false>)); DVT_MAX_SHARED((fit_loss_kernel<6, true>));
  DVT_MAX_SHARED((fit_loss_kernel<8, false>)); DVT_MAX_SHARED((fit_loss_kernel<8, true>));
  DVT_MAX_SHARED((fit_loss_kernel<12, false>)); DVT_MAX_SHARED((fit_loss_kernel<12, true>));
#undef DVT_MAX_SHARED
  return DVT_OK;
}

static int fit_alloc(Fit* f, void** p, size_t bytes, bool zero = true) {
  DVT_CUDA_OK(cudaMalloc(p, bytes));
  f->owned.push_back(*p);
  if (zero) DVT_CUDA_OK(cudaMemset(*p, 0, bytes));
  return DVT_OK;
}

static int r8(int x) { return (x + 7) / 8 * 8; }

int fit_create(Fit** out, int C, int gh, int gw, int bsz, int n_levels, const float* scale, const uint32_t* res,
               const uint32_t* size, const uint32_t* offset, const uint32_t* hashed) {
  DVT_REQUIRE(C % 32 == 0 && C >= 32 && C <= 1536, "fit: feat_dim %d unsupported (multiple of 32, <= 1536)", C);
  DVT_REQUIRE(n_levels >= 1 && n_levels <= FIT_MAX_LEVELS, "fit: n_levels %d out of range", n_levels);
  DVT_REQUIRE(bsz >= 8 && bsz % 8 == 0, "fit: pixel batch %d must be a positive multiple of 8", bsz);
  DVT_REQUIRE(gh > 0 && gw > 0, "fit: bad noise-map size");
  {
    int prc = gemm_prepare();
    if (prc) return prc;
    prc = fit_prepare_kernels();
    if (prc) return prc;
  }
  // DVT_FIT_SWEEP_STEPS="k1[,k2]" per phase: the pipelined sweep makes one pass over the table per window of k steps
  // (1 <= k <= FIT_MAX_WINDOW; 1 = one pass per step).  The sequential schedule sweeps every step.
  int win[2] = {Fit().sweep_steps[0], Fit().sweep_steps[1]};
  if (const char* ss = getenv("DVT_FIT_SWEEP_STEPS")) {
    const int got = sscanf(ss, "%d,%d", &win[0], &win[1]);
    if (got == 1) win[1] = win[0];
    DVT_REQUIRE(got >= 1, "fit: DVT_FIT_SWEEP_STEPS '%s' is not \"k1[,k2]\"", ss);
  }
  for (int q = 0; q < 2; ++q)
    DVT_REQUIRE(win[q] >= 1 && win[q] <= FIT_MAX_WINDOW, "fit: DVT_FIT_SWEEP_STEPS %d out of range [1, %d]", win[q],
                FIT_MAX_WINDOW);
  Fit* f = new Fit();
  int prio_lo = 0, prio_hi = 0;  // (numerically lower = higher priority)
  DVT_CUDA_OK(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
  DVT_CUDA_OK(cudaStreamCreateWithPriority(&f->stream, cudaStreamNonBlocking, prio_hi));
  DVT_CUDA_OK(cudaStreamCreateWithPriority(&f->sB, cudaStreamNonBlocking, prio_hi));
  DVT_CUDA_OK(cudaStreamCreateWithPriority(&f->sC, cudaStreamNonBlocking, prio_hi));
  DVT_CUDA_OK(cudaStreamCreateWithPriority(&f->sE, cudaStreamNonBlocking, prio_hi));
  DVT_CUDA_OK(cudaStreamCreateWithPriority(&f->sD, cudaStreamNonBlocking, prio_lo));  // the sweep yields to the chain
  DVT_CUDA_OK(cudaStreamCreateWithFlags(&f->sU, cudaStreamNonBlocking));
  for (auto& e : f->ev_upload) DVT_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto& e : f->ev_run_done) DVT_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto& e : f->ev) DVT_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  for (auto& e : f->ev_sweep) DVT_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  DVT_CUDA_OK(cudaEventCreateWithFlags(&f->ev_in, cudaEventDisableTiming));
  DVT_CUDA_OK(cudaEventCreateWithFlags(&f->ev_out, cudaEventDisableTiming));
  {
    // Schedule knobs (defaults chosen at the headline size; not yet re-tuned for the 132 SMs of an H100):
    //   DVT_FIT_SWEEP_CTAS="a[,b]"  per phase (1 [, 2]): n > 0 pipelined sweep on n persistent CTAs (1024 threads, one
    //                               per SM); 0 pipelined sweep on 8 x #SM CTAs of 256 threads; -1 sequential schedule
    //   DVT_FIT_PIPELINE=0          sequential schedule in both phases
    int cfg[2] = {48, 48};
    if (const char* se = getenv("DVT_FIT_SWEEP_CTAS")) {
      int a = 0, b = 0;
      const int got = sscanf(se, "%d,%d", &a, &b);
      if (got >= 1) { cfg[0] = a; cfg[1] = got >= 2 ? b : a; }
    }
    //   DVT_FIT_PDL=0               plain stream-ordered launches (no programmatic dependent launch)
    //   DVT_FIT_RES_TF32=1          residual-MLP GEMMs in plain TF32 instead of 3xTF32 (experiment; not the default)
    //   DVT_FIT_SWEEP_TMA=1         persistent sweep CTAs use the TMA-staged kernel instead of plain loads (bit-identical;
    //                               kept as a tested experiment)
    const char* tm = getenv("DVT_FIT_SWEEP_TMA");
    f->sweep_tma = tm && tm[0] == '1';
    //   DVT_FIT_WGRAD_TF32=1        weight-gradient GEMMs of the field MLP in plain TF32 (experiment; not the default)
    const char* wt = getenv("DVT_FIT_WGRAD_TF32");
    f->wgrad_x3 = (wt && wt[0] == '1') ? 2 : 1;
    //   DVT_FIT_SWEEP_PDL=0         sweep t+1 is launched only when sweep t has completed (no waiting resident CTAs)
    //   DVT_FIT_X3_WIDE_MIN_N="a[,b]" per phase: 3xTF32 GEMMs with N >= this use 128 x 128 tiles (0: always 128 x 64)
    //   DVT_FIT_WGRAD_SMS=n         split-K of the weight-gradient GEMMs fills at most n SMs (they share the GPU with the
    //                               data-gradient GEMMs of the critical path)
    //   DVT_FIT_OFFPATH_PRIO=n      launch priority of the kernels that only feed Adam(small), n levels below the chain.
    //                               The graphs keep the attribute (DVT_FIT_DEBUG_GRAPH=1 shows it).  Default 0.
    if (const char* sp_ = getenv("DVT_FIT_SWEEP_PDL")) f->sweep_pdl = sp_[0] != '0';
    if (const char* wm = getenv("DVT_FIT_X3_WIDE_MIN_N")) {
      int a = 0, b = 0;
      const int got = sscanf(wm, "%d,%d", &a, &b);
      if (got >= 1) f->x3_wide_min_n[0] = f->x3_wide_min_n[1] = std::max(0, a);
      if (got == 2) f->x3_wide_min_n[1] = std::max(0, b);
    }
    if (const char* st_ = getenv("DVT_FIT_SWEEP_THREADS")) f->sweep_threads = std::min(1024, std::max(128, atoi(st_) / 32 * 32));
    if (const char* ws = getenv("DVT_FIT_WGRAD_SMS")) f->wgrad_sms = std::max(1, atoi(ws));
    if (const char* op = getenv("DVT_FIT_OFFPATH_PRIO")) f->off_path_prio_drop = std::max(0, atoi(op));
    const char* rt = getenv("DVT_FIT_RES_TF32");
    f->res_x3 = (rt && rt[0] == '1') ? 2 : 1;
    const char* pd = getenv("DVT_FIT_PDL");
    f->pdl = !(pd && pd[0] == '0');
    const char* pe = getenv("DVT_FIT_PIPELINE");
    const bool off = pe && pe[0] == '0';
    for (int q = 0; q < 2; ++q) {
      f->pipe[q] = !off && cfg[q] >= 0;
      f->sweep_ctas[q] = f->pipe[q] ? std::min(cfg[q], num_sms()) : 0;
    }
    for (int q = 0; q < 2; ++q) f->sweep_steps[q] = f->pipe[q] ? win[q] : 1;
  }
  f->C = C; f->gh = gh; f->gw = gw; f->hw = gh * gw; f->bsz = bsz; f->Lf = n_levels * FIT_F;
  f->grid.n_levels = n_levels;
  for (int l = 0; l < n_levels; ++l) {
    f->grid.scale[l] = scale[l]; f->grid.res[l] = res[l]; f->grid.size[l] = size[l];
    f->grid.offset[l] = offset[l]; f->grid.hashed[l] = hashed[l];
  }
  f->grid.offset[n_levels] = offset[n_levels];
  f->n_table = (size_t)offset[n_levels] * FIT_F;
  int off = 0;
  auto seg = [&](Seg& s, int rows, int cols) { s.off = off; s.rows = rows; s.cols = cols; off += r8(rows * cols); };
  const int H1 = C / 2, Hr = C / 4;
  seg(f->W1, H1, f->Lf); seg(f->b1, H1, 1); seg(f->W2, C, H1); seg(f->b2, C, 1);
  seg(f->G, f->hw, C);
  seg(f->R1, Hr, C); seg(f->rb1, Hr, 1); seg(f->R2, Hr, Hr); seg(f->rb2, Hr, 1); seg(f->R3, C, Hr); seg(f->rb3, C, 1);
  f->n_small = off;
  f->ld_enc = f->Lf + 8; f->ld_h1 = H1 + 8; f->ld_raw = C + 8; f->ld_r = Hr + 8;
  int rc = 0;
  auto A = [&](void** p, size_t bytes) { if (!rc) rc = fit_alloc(f, p, bytes); };
  for (int q = 0; q < 2; ++q) {
    A((void**)&f->tb.p[q], f->n_table * 4); A((void**)&f->tb.m[q], f->n_table * 4); A((void**)&f->tb.v[q], f->n_table * 4);
  }
  // Gradient ring: the backward of step t (window u) overwrites slot t % ring, last used by step t - ring.  Window u's
  // first backward waits for the sweep of window u - 2, and every reader of a step's gradient (its window's sweep, the
  // encodes of its window and of the next one) is done by then; with windows of at most k steps, t - 2k lies before
  // window u - 1, so 2k slots suffice.
  f->tb.ring = 2 * std::max(f->sweep_steps[0], f->sweep_steps[1]);
  f->tb.n_entries = f->n_table / FIT_F;
  A((void**)&f->tb.g, f->tb.ring * f->n_table * 4);
  A((void**)&f->tb.stamp, f->tb.ring * f->tb.n_entries * 4);
  A((void**)&f->sp, (size_t)off * 4); A((void**)&f->sm, (size_t)off * 4); A((void**)&f->sv, (size_t)off * 4);
  A((void**)&f->sg, (size_t)off * 4); A((void**)&f->wsplit, (size_t)off * 8);
  const size_t n = bsz;
  A((void**)&f->enc, n * f->ld_enc * 8); A((void**)&f->h1, n * f->ld_h1 * 8); A((void**)&f->dpred, n * C * 8);
  A((void**)&f->dh1, n * H1 * 8); A((void**)&f->Fout, n * C * 4); A((void**)&f->denc, n * f->Lf * 4);
  A((void**)&f->rawb, n * f->ld_raw * 8); A((void**)&f->r1, n * f->ld_r * 8); A((void**)&f->r2, n * f->ld_r * 8);
  A((void**)&f->dR, n * C * 8); A((void**)&f->dr2, n * Hr * 8); A((void**)&f->dr1, n * Hr * 8);
  A((void**)&f->Rout, n * C * 4); A((void**)&f->step_base, 2 * sizeof(int));
  A((void**)&f->inputs_dev, sizeof(FitInputs));
  A((void**)&f->flags_dev, sizeof(int));
  A((void**)&f->wg_sem, 5 * FIT_SEM_TILES * sizeof(unsigned));
  if (!rc && cudaHostAlloc((void**)&f->flags_pinned, sizeof(int), cudaHostAllocDefault) != cudaSuccess) rc = DVT_ERR_CUDA;
  if (rc) { for (void* p : f->owned) cudaFree(p); delete f; return rc; }
  // ones columns (bias gradients through the weight-gradient GEMMs)
  const int tb = 256, nb = (bsz + tb - 1) / tb;
  fit_fill_col_kernel<<<nb, tb>>>(f->enc, f->ld_enc, f->Lf, bsz, 1.f);
  fit_fill_col_kernel<<<nb, tb>>>(f->h1, f->ld_h1, H1, bsz, 1.f);
  fit_fill_col_kernel<<<nb, tb>>>(f->rawb, f->ld_raw, C, bsz, 1.f);
  fit_fill_col_kernel<<<nb, tb>>>(f->r1, f->ld_r, Hr, bsz, 1.f);
  fit_fill_col_kernel<<<nb, tb>>>(f->r2, f->ld_r, Hr, bsz, 1.f);
  DVT_CUDA_OK(cudaDeviceSynchronize());
  *out = f;
  return DVT_OK;
}

static void fit_drop_graphs(Fit* f) {
  if (f->graph1) cudaGraphExecDestroy(f->graph1);
  if (f->graph2) cudaGraphExecDestroy(f->graph2);
  f->graph1 = f->graph2 = nullptr;
}

void fit_destroy(Fit* f) {
  if (!f) return;
  fit_drop_graphs(f);
  if (f->stream) cudaStreamDestroy(f->stream);
  if (f->sB) cudaStreamDestroy(f->sB);
  if (f->sC) cudaStreamDestroy(f->sC);
  if (f->sE) cudaStreamDestroy(f->sE);
  if (f->sD) cudaStreamDestroy(f->sD);
  if (f->sU) cudaStreamDestroy(f->sU);
  for (auto& e : f->ev_upload) if (e) cudaEventDestroy(e);
  for (auto& e : f->ev_run_done) if (e) cudaEventDestroy(e);
  for (auto& e : f->ev) if (e) cudaEventDestroy(e);
  for (auto& e : f->ev_sweep) if (e) cudaEventDestroy(e);
  if (f->ev_in) cudaEventDestroy(f->ev_in);
  if (f->ev_out) cudaEventDestroy(f->ev_out);
  for (void* p : f->owned) cudaFree(p);
  for (int q = 0; q < 2; ++q) { cudaFree(f->idx[q]); cudaFreeHost(f->idx_pinned[q]); }
  cudaFreeHost(f->flags_pinned);
  cudaFree(f->sc_main); cudaFree(f->sc_res); cudaFree(f->losses);
  cudaFree(f->q_enc); cudaFree(f->q_h1); cudaFree(f->q_raw); cudaFree(f->q_r1); cudaFree(f->q_r2); cudaFree(f->q_stage);
  delete f;
}

static bool fit_find(Fit* f, const std::string& name, Seg** s) {
  struct { const char* n; Seg* s; } tab[] = {
      {"mlp.0.weight", &f->W1}, {"mlp.0.bias", &f->b1}, {"mlp.2.weight", &f->W2}, {"mlp.2.bias", &f->b2},
      {"G", &f->G}, {"res.0.weight", &f->R1}, {"res.0.bias", &f->rb1}, {"res.2.weight", &f->R2},
      {"res.2.bias", &f->rb2}, {"res.4.weight", &f->R3}, {"res.4.bias", &f->rb3}};
  for (auto& t : tab)
    if (name == t.n) { *s = t.s; return true; }
  return false;
}

static int fit_stage(Fit* f, size_t floats) {
  if (f->q_stage_cap < floats) {
    cudaFree(f->q_stage); f->q_stage = nullptr; f->q_stage_cap = 0;
    DVT_CUDA_OK(cudaMalloc(&f->q_stage, floats * 4));
    f->q_stage_cap = floats;
  }
  return DVT_OK;
}

// ----------------------------------------------------------------------------------------------------
// Stream discipline of the host engine.  Every call that MUTATES engine state (init / set_param / begin / run) first makes
// the engine's main stream wait for the caller's stream and enqueues its device work on the engine's stream; every call
// that READS state on the caller's stream (query / residual / losses / get_param) first makes the caller's stream wait for
// the engine's.  Nothing in between synchronises the host with the device, so a driver can enqueue image i+1 while image
// i is still being fitted (Stage1Pipeline.run_images).
// ----------------------------------------------------------------------------------------------------
static int fit_after_caller(Fit* f, cudaStream_t caller) {
  DVT_CUDA_OK(cudaEventRecord(f->ev_in, caller));
  DVT_CUDA_OK(cudaStreamWaitEvent(f->stream, f->ev_in, 0));
  return DVT_OK;
}
static int fit_before_caller(Fit* f, cudaStream_t caller) {
  DVT_CUDA_OK(cudaEventRecord(f->ev_out, f->stream));
  DVT_CUDA_OK(cudaStreamWaitEvent(caller, f->ev_out, 0));
  return DVT_OK;
}

// Parameter names follow oracle/fit.py::PARAM_ORDER ("G" is the reference's shared_artifacts [1, C, h, w]).
// src: host or device memory.  Device sources may be temporaries of the caller's stream-ordered allocator: the caller's
// stream is made to wait for the copy, so the memory is not reused before it has been read.
int fit_set_param(Fit* f, const char* name_c, const float* src, size_t numel, cudaStream_t caller) {
  const std::string name(name_c);
  Seg* s = nullptr;
  if (name != "table") {
    DVT_REQUIRE(fit_find(f, name, &s), "fit_set_param: unknown parameter %s", name_c);
    const size_t expect = (size_t)s->rows * s->cols;
    DVT_REQUIRE(numel == expect, "fit_set_param: %s has %zu elements, expected %zu", name_c, numel, expect);
  } else {
    DVT_REQUIRE(numel == f->n_table, "fit_set_param: table has %zu elements, expected %zu", numel, f->n_table);
  }
  int rc = fit_after_caller(f, caller);
  if (rc) return rc;
  cudaStream_t st = f->stream;
  if (name == "table") {
    DVT_CUDA_OK(cudaMemcpyAsync(f->tb.p[f->cur_buf], src, numel * 4, cudaMemcpyDefault, st));
  } else if (name == "G") {  // [C, h*w] -> [h*w, C]
    if (f->q_stage_cap < numel) DVT_CUDA_OK(cudaStreamSynchronize(st));  // the staging buffer is about to be replaced
    rc = fit_stage(f, numel);
    if (rc) return rc;
    DVT_CUDA_OK(cudaMemcpyAsync(f->q_stage, src, numel * 4, cudaMemcpyDefault, st));
    fit_transpose_kernel<<<256, 256, 0, st>>>(f->q_stage, f->sp + s->off, f->C, f->hw);
    DVT_CUDA_OK(cudaGetLastError());
  } else {
    DVT_CUDA_OK(cudaMemcpyAsync(f->sp + s->off, src, numel * 4, cudaMemcpyDefault, st));
    // the GEMMs read the weights as TF32 hi / lo planes: keep them current (fit_query / fit_residual may follow directly)
    fit_split_kernel<<<64, 256, 0, st>>>(f->sp + s->off, f->wsplit + s->off, numel, (size_t)f->n_small);
    DVT_CUDA_OK(cudaGetLastError());
  }
  return fit_before_caller(f, caller);
}

int fit_get_param(Fit* f, const char* name_c, float* dst, size_t numel) {
  const std::string name(name_c);
  DVT_CUDA_OK(cudaDeviceSynchronize());
  // "table.next": the buffer a sweep writes (dvt_fit_sweep_once, tests); "table.m" / "table.v": the table's Adam moments
  if (name == "table" || name == "table.next" || name == "table.m" || name == "table.v") {
    DVT_REQUIRE(numel == f->n_table, "fit_get_param: table size mismatch");
    const int b = f->cur_buf ^ (name == "table.next" ? 1 : 0);
    const float* src = name == "table.m" ? f->tb.m[b] : name == "table.v" ? f->tb.v[b] : f->tb.p[b];
    DVT_CUDA_OK(cudaMemcpy(dst, src, numel * 4, cudaMemcpyDefault));
    return DVT_OK;
  }
  Seg* s = nullptr;
  DVT_REQUIRE(fit_find(f, name, &s), "fit_get_param: unknown parameter %s", name_c);
  DVT_REQUIRE(numel == (size_t)s->rows * s->cols, "fit_get_param: %s size mismatch", name_c);
  if (name == "G") {
    int rc = fit_stage(f, numel);
    if (rc) return rc;
    fit_transpose_kernel<<<256, 256>>>(f->sp + s->off, f->q_stage, f->hw, f->C);
    DVT_CUDA_OK(cudaGetLastError());
    DVT_CUDA_OK(cudaMemcpy(dst, f->q_stage, numel * 4, cudaMemcpyDefault));
  } else {
    DVT_CUDA_OK(cudaMemcpy(dst, f->sp + s->off, numel * 4, cudaMemcpyDefault));
  }
  return DVT_OK;
}

// Installs the per-node tables of F.grid_sample(G, linspace(-1, 1) nodes, align_corners=True) (see LossArgs): HOST arrays
// of gw + gh entries (x nodes first).  The caller computes them with the reference's own fp32 arithmetic
// (dvt/fit.py::artifact_axis_table).  Changes the step kernels' arguments: captured graphs are dropped.
int fit_set_artifact_grid(Fit* f, const int* i0, const float* w0, const float* w1) {
  DVT_REQUIRE(i0 && w0 && w1, "fit_set_artifact_grid: null argument");
  const size_t n = (size_t)f->gw + f->gh;
  DVT_CUDA_OK(cudaDeviceSynchronize());
  fit_drop_graphs(f);
  if (!f->ax_i0) {
    int rc = fit_alloc(f, (void**)&f->ax_i0, n * 4);
    if (!rc) rc = fit_alloc(f, (void**)&f->ax_w0, n * 4);
    if (!rc) rc = fit_alloc(f, (void**)&f->ax_w1, n * 4);
    if (rc) return rc;
  }
  DVT_CUDA_OK(cudaMemcpy(f->ax_i0, i0, n * 4, cudaMemcpyHostToDevice));
  DVT_CUDA_OK(cudaMemcpy(f->ax_w0, w0, n * 4, cudaMemcpyHostToDevice));
  DVT_CUDA_OK(cudaMemcpy(f->ax_w1, w1, n * 4, cudaMemcpyHostToDevice));
  return DVT_OK;
}

// ---- device-side (re-)initialisation of all parameters: what constructing fresh SingleImageDenoiser /
// NeuralFeatureField modules does in the reference for every image (main_img_denoising.py:39-47), without a host round
// trip.  Counter-based generator: element e of tensor `tid` under `seed` is a pure function of (seed, tid, e).
__device__ __forceinline__ uint64_t mix64(uint64_t z) {  // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ float u01(uint64_t seed, uint32_t tid, uint64_t e, uint32_t draw) {
  const uint64_t h = mix64(mix64(seed + 0x9E3779B97F4A7C15ull * (tid + 1)) ^ (e * 2 + draw + 0x632BE59BD9B4E019ull));
  return (float)((h >> 40) + 1) * (1.0f / 16777217.0f);  // (0, 1)
}
// kind 0: U(-bound, bound); kind 1: N(0, 1) * bound (Box-Muller); kind 2: U(-bound, bound) stored transposed: element
// e = c * cols + r of a [rows?]... (G is drawn in the reference's [C, h*w] order and stored [h*w, C])
__global__ void fit_init_kernel(float* __restrict__ dst, size_t n, uint64_t seed, uint32_t tid, int kind, float bound,
                                int t_rows, int t_cols) {
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
    float val;
    if (kind == 1) {
      const float u1 = u01(seed, tid, e, 0), u2 = u01(seed, tid, e, 1);
      val = sqrtf(-2.0f * logf(u1)) * cospif(2.0f * u2) * bound;
    } else {
      val = (2.0f * u01(seed, tid, e, 0) - 1.0f) * bound;
    }
    size_t o = e;
    if (t_rows > 0) {  // e indexes [t_rows, t_cols]; stored transposed
      const size_t r = e / t_cols, c = e - r * t_cols;
      o = c * t_rows + r;
    }
    dst[o] = val;
  }
}

// Fresh parameters for the next fit: hash table U(-1e-4, 1e-4) (tcnn's default grid initialisation), nn.Linear default
// initialisation U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for all MLP weights and biases, G = randn * 0.02
// (offline_denoiser.py:33-36).  The reference's own streams (tcnn pcg32, torch's Philox) are not reproduced -- no test of
// the reference pins them -- but the distributions are.
int fit_init_params(Fit* f, uint64_t seed, cudaStream_t caller) {
  int rc = fit_after_caller(f, caller);
  if (rc) return rc;
  cudaStream_t st = f->stream;
  auto launch = [&](float* dst, size_t n, uint32_t tid, int kind, float bound, int tr = 0, int tc = 0) -> int {
    const int blocks = (int)std::min<size_t>((n + 255) / 256, (size_t)num_sms() * 8);
    fit_init_kernel<<<blocks, 256, 0, st>>>(dst, n, seed, tid, kind, bound, tr, tc);
    DVT_CUDA_OK(cudaGetLastError());
    count_launch();
    return DVT_OK;
  };
  f->cur_host = 0;
  f->cur_buf = 0;
  FIT_RC0(launch(f->tb.p[0], f->n_table, 0, 0, 1e-4f));
  struct { Seg* w; Seg* b; uint32_t tid; } lin[] = {{&f->W1, &f->b1, 1}, {&f->W2, &f->b2, 3}, {&f->R1, &f->rb1, 5},
                                                    {&f->R2, &f->rb2, 7}, {&f->R3, &f->rb3, 9}};
  for (auto& l : lin) {
    const float bound = 1.0f / sqrtf((float)l.w->cols);
    FIT_RC0(launch(f->sp + l.w->off, (size_t)l.w->rows * l.w->cols, l.tid, 0, bound));
    FIT_RC0(launch(f->sp + l.b->off, (size_t)l.b->rows, l.tid + 1, 0, bound));
  }
  FIT_RC0(launch(f->sp + f->G.off, (size_t)f->hw * f->C, 11, 1, 0.02f, f->C, f->hw));
  fit_split_kernel<<<256, 256, 0, st>>>(f->sp, f->wsplit, (size_t)f->n_small, (size_t)f->n_small);
  DVT_CUDA_OK(cudaGetLastError());
  return fit_before_caller(f, caller);
}

// clamps out-of-range sampled rows (so that no kernel can read outside the bank) and records what it saw
__global__ void fit_check_inputs_kernel(const float* __restrict__ coords, size_t n2, int* __restrict__ idx, size_t n_idx,
                                        int bank_rows, int* __restrict__ flags) {
  int bad = 0;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n2; e += stride) {
    const float c = coords[e];
    if (!(c >= 0.f && c <= 1.f)) bad |= 1;
  }
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n_idx; e += stride) {
    const int v = idx[e];
    if (v < 0 || v >= bank_rows) {
      bad |= 2;
      idx[e] = min(max(v, 0), bank_rows - 1);
    }
  }
  if (bad) atomicOr(flags, bad);
}

__global__ void fit_set_inputs_kernel(FitInputs* dst, const float* bank, const float* coords, const int* idx,
                                      int* step_base) {
  dst->bank = bank;
  dst->coords = coords;
  dst->idx = idx;
  step_base[0] = 0;
  step_base[1] = 0;
}

static int fit_flags_to_error(int flags) {
  DVT_REQUIRE((flags & 1) == 0, "coordinates should be in [0, 1]");
  DVT_REQUIRE((flags & 2) == 0, "fit_begin: a sampled bank row is out of range");
  return DVT_OK;
}

// Reads the input-validation flags of the fits begun since the last check (blocks until the engine's stream is idle).
int fit_check(Fit* f) {
  DVT_CUDA_OK(cudaMemcpyAsync(f->flags_pinned, f->flags_dev, sizeof(int), cudaMemcpyDeviceToHost, f->stream));
  DVT_CUDA_OK(cudaMemsetAsync(f->flags_dev, 0, sizeof(int), f->stream));
  DVT_CUDA_OK(cudaStreamSynchronize(f->stream));
  return fit_flags_to_error(*f->flags_pinned);
}

// Starts a fit: zeroes the optimiser state / gradients, rebuilds the TF32 operand planes of the weights and installs the
// bank, the sampling stream and the schedule.  Everything is enqueued; nothing waits for the device unless `validate`
// (then the range checks are read back and reported here, like the reference's assert, neural_feature_field.py:47).
// idx_host: int32 [num_iters, bsz] bank rows (the np.random.randint stream, main_img_denoising.py:73).
int fit_begin(Fit* f, const float* bank, const float* coords, size_t bank_rows, const int* idx_host, int num_iters,
              double lr, double min_lr, int warmup_iters, int freeze_step, double weight_decay, double loss_scale,
              int validate, cudaStream_t caller) {
  DVT_REQUIRE(bank && coords && idx_host && num_iters > 0, "fit_begin: bad arguments");
  DVT_REQUIRE(bank_rows % (size_t)f->hw == 0, "fit_begin: bank rows %zu not a multiple of h*w = %d", bank_rows, f->hw);
  DVT_REQUIRE(bank_rows < (size_t)1 << 31, "fit_begin: bank of %zu rows exceeds the int32 row index", bank_rows);
  DVT_REQUIRE(freeze_step >= 0, "fit_begin: negative freeze step");
  f->bank = bank; f->coords = coords; f->bank_rows = bank_rows;
  // scalars that are baked into captured kernel nodes
  if (f->wd != (float)weight_decay || f->loss_scale != (float)loss_scale || freeze_step != f->freeze_step) {
    DVT_CUDA_OK(cudaStreamSynchronize(f->stream));
    fit_drop_graphs(f);
  }
  f->wd = (float)weight_decay; f->loss_scale = (float)loss_scale;
  const size_t n_idx = (size_t)num_iters * f->bsz;
  // ---- rare path: buffers sized by the schedule length ----
  if (n_idx + f->bsz > f->idx_cap) {
    DVT_CUDA_OK(cudaDeviceSynchronize());
    for (int q = 0; q < 2; ++q) {
      cudaFree(f->idx[q]); cudaFreeHost(f->idx_pinned[q]);
      f->idx[q] = nullptr; f->idx_pinned[q] = nullptr;
      DVT_CUDA_OK(cudaMalloc(&f->idx[q], (n_idx + f->bsz) * 4));
      DVT_CUDA_OK(cudaHostAlloc((void**)&f->idx_pinned[q], n_idx * 4, cudaHostAllocDefault));
      f->run_done_valid[q] = false;
    }
    f->idx_cap = n_idx + f->bsz;
  }
  if (num_iters != f->num_iters) {
    DVT_CUDA_OK(cudaDeviceSynchronize());
    cudaFree(f->sc_main); cudaFree(f->sc_res); cudaFree(f->losses);
    f->sc_main = f->sc_res = nullptr; f->losses = nullptr;
    DVT_CUDA_OK(cudaMalloc(&f->sc_main, (size_t)(num_iters + 1) * sizeof(AdamScalars)));
    DVT_CUDA_OK(cudaMalloc(&f->sc_res, (size_t)(num_iters + 1) * sizeof(AdamScalars)));
    DVT_CUDA_OK(cudaMalloc(&f->losses, (size_t)num_iters * 5 * 4));
    f->sched_key[0] = -1;
    fit_drop_graphs(f);
  }
  f->num_iters = num_iters; f->freeze_step = freeze_step; f->cur_step = 0;
  // ---- sampling stream: staged through pinned memory and copied on the upload stream, beside the running fit ----
  const int slot = f->idx_slot ^ 1;
  f->idx_slot = slot;
  DVT_CUDA_OK(cudaEventSynchronize(f->ev_upload[slot]));  // the copy that last read this staging buffer (long done)
  memcpy(f->idx_pinned[slot], idx_host, n_idx * 4);
  if (f->run_done_valid[slot]) DVT_CUDA_OK(cudaStreamWaitEvent(f->sU, f->ev_run_done[slot], 0));  // its last reader
  DVT_CUDA_OK(cudaMemcpyAsync(f->idx[slot], f->idx_pinned[slot], n_idx * 4, cudaMemcpyHostToDevice, f->sU));
  DVT_CUDA_OK(cudaMemsetAsync(f->idx[slot] + n_idx, 0, (size_t)f->bsz * 4, f->sU));  // rows of the (unused) encode of step num_iters
  DVT_CUDA_OK(cudaEventRecord(f->ev_upload[slot], f->sU));
  // ---- schedule tables (dvt/utils/misc.py:306-322), cached: they depend on the hyper-parameters only ----
  const double key[6] = {(double)num_iters, (double)warmup_iters, lr, min_lr, (double)freeze_step, 1.0};
  if (memcmp(key, f->sched_key, sizeof(key)) != 0) {
    std::vector<AdamScalars> a(num_iters + 1), b(num_iters + 1);
    for (int s = 0; s <= num_iters; ++s) {
      double lrs;
      if (s < warmup_iters) lrs = lr * s / warmup_iters;
      else lrs = min_lr + (lr - min_lr) * 0.5 * (1.0 + cos(M_PI * (s - warmup_iters) / (double)(num_iters - warmup_iters)));
      const int t = s + 1;
      a[s].step_size = (float)(lrs / (1.0 - pow(0.9, t)));
      a[s].inv_bc2_sqrt = (float)(1.0 / sqrt(1.0 - pow(0.99, t)));
      const int tr = s - freeze_step;  // residual MLP: first update at s = freeze_step + 1 has t = 1
      if (tr >= 1) {
        b[s].step_size = (float)(lrs / (1.0 - pow(0.9, tr)));
        b[s].inv_bc2_sqrt = (float)(1.0 / sqrt(1.0 - pow(0.99, tr)));
      } else {
        b[s].step_size = 0.f; b[s].inv_bc2_sqrt = 1.f;
      }
    }
    DVT_CUDA_OK(cudaStreamSynchronize(f->stream));  // a running fit still reads the old tables
    DVT_CUDA_OK(cudaMemcpy(f->sc_main, a.data(), a.size() * sizeof(AdamScalars), cudaMemcpyHostToDevice));
    DVT_CUDA_OK(cudaMemcpy(f->sc_res, b.data(), b.size() * sizeof(AdamScalars), cudaMemcpyHostToDevice));
    memcpy(f->sched_key, key, sizeof(key));
  }
  // ---- device state, in stream order behind the previous fit and the caller's pending work ----
  int rc = fit_after_caller(f, caller);
  if (rc) return rc;
  cudaStream_t st = f->stream;
  DVT_CUDA_OK(cudaStreamWaitEvent(st, f->ev_upload[slot], 0));
  fit_set_inputs_kernel<<<1, 1, 0, st>>>(f->inputs_dev, bank, coords, f->idx[slot], f->step_base);
  fit_check_inputs_kernel<<<256, 256, 0, st>>>(coords, bank_rows * 2, f->idx[slot], n_idx, (int)bank_rows, f->flags_dev);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch(2);
  DVT_CUDA_OK(cudaMemsetAsync(f->losses, 0, (size_t)num_iters * 5 * 4, st));
  if (f->cur_buf)  // the schedule restarts with no sweep done: its state lives in buffer 0
    DVT_CUDA_OK(cudaMemcpyAsync(f->tb.p[0], f->tb.p[1], f->n_table * 4, cudaMemcpyDeviceToDevice, st));
  f->cur_host = 0;
  f->cur_buf = 0;
  DVT_CUDA_OK(cudaMemsetAsync(f->tb.m[0], 0, f->n_table * 4, st));
  DVT_CUDA_OK(cudaMemsetAsync(f->tb.v[0], 0, f->n_table * 4, st));
  // stamps of the previous fit would match this one's steps; the gradient slots need no reset (a step's first touch
  // of an entry overwrites, fit_grid_bwd_kernel)
  DVT_CUDA_OK(cudaMemsetAsync(f->tb.stamp, 0, (size_t)f->tb.ring * f->tb.n_entries * 4, st));
  f->enc_ready = false;
  f->epoch_steps = f->epoch_windows = f->win_first = f->prev_first = 0;
  f->epoch_forked = false;
  DVT_CUDA_OK(cudaMemsetAsync(f->sm, 0, (size_t)f->n_small * 4, st));
  DVT_CUDA_OK(cudaMemsetAsync(f->sv, 0, (size_t)f->n_small * 4, st));
  DVT_CUDA_OK(cudaMemsetAsync(f->sg, 0, (size_t)f->n_small * 4, st));
  fit_split_kernel<<<256, 256, 0, st>>>(f->sp, f->wsplit, (size_t)f->n_small, (size_t)f->n_small);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  if (validate) return fit_check(f);
  return DVT_OK;
}

#define FIT_RC(x) do { int _rc = (x); if (_rc) return _rc; } while (0)

// GEMM operands of the fit are fp32 hi/lo plane pairs; all products are 3xTF32 (fp32-accurate, gemm.cu "x3").
struct Op {
  const float* p;
  int ld;
  size_t plane;
};

// Y = act(X W^T + b):  X [M, K] planes, W [N, K] planes.  split_out: Y is written as hi/lo planes (feeds a GEMM).
static int fit_linear(Op X, int M, int K, Op W, int N, const float* bias, int act, float* out, int ldo, size_t out_plane,
                      bool split_out, cudaStream_t st, int impl, bool pdl = false, int x3 = 1, int prio_drop = 0,
                      int wide = 0) {
  GemmEpi e;
  e.bias = bias; e.act = act; e.out = out; e.ldo = ldo; e.out_plane = out_plane;
  e.out_mode = split_out ? OUT_F32_SPLIT : OUT_F32;
  GemmShape s{M, N, K, 1};
  s.x3 = x3; s.plane_a = X.plane; s.plane_b = W.plane; s.pdl = pdl; s.prio_drop = prio_drop; s.x3_wide_min_n = wide;
  return launch_gemm_tn(X.p, X.ld, W.p, W.ld, TMAP_F32, s, e, st, impl);
}

// dX = (dY . W) * (H > 0):  dY [M, Nout] K-major A; W stored [Nout, Kin] = MN-major B with N = Kin
static int fit_dgrad(Op dY, int M, int Nout, Op W, int Kin, const float* Hmask, int ldmask, float* out, int ldo,
                     size_t out_plane, bool split_out, cudaStream_t st, int impl, bool pdl = false, int x3 = 1,
                     int prio_drop = 0, int wide = 0) {
  GemmEpi e;
  e.mask_f32 = Hmask; e.ldmask = ldmask; e.out = out; e.ldo = ldo; e.out_plane = out_plane;
  e.out_mode = split_out ? OUT_F32_SPLIT : OUT_F32;
  GemmShape s{M, Kin, Nout, 1};
  s.b_mn = 1; s.x3 = x3; s.plane_a = dY.plane; s.plane_b = W.plane; s.pdl = pdl; s.prio_drop = prio_drop; s.x3_wide_min_n = wide;
  return launch_gemm_tn(dY.p, dY.ld, W.p, W.ld, TMAP_F32, s, e, st, impl);
}

// dW[Nout, Kin] (+ db[Nout]) += dY^T . [X | 1]:  dY stored [n, Nout] (MN-major A), X stored [n, Kin + ones] (MN-major B)
// sem: FIT_SEM_TILES zeroed per-tile counters of this call site: the splits of a tile add their partial sums in split
// order, so the gradient does not depend on which split finishes first.
static int fit_wgrad(Op dY, int n, int Nout, Op X, int Kin, float* gW, float* gb, unsigned* sem, cudaStream_t st, int impl,
                     bool pdl = false, int x3 = 1, int prio_drop = 0, int wide = 0, int sm_cap = 1 << 20) {
  GemmEpi e;
  e.out = gW; e.ldo = Kin; e.out_mode = OUT_F32_ATOMIC; e.last_col_out = gb; e.splitk_sem = sem;
  // split-K so that (output tiles x splits) fills the SMs once: tiles are 128 x 64 or 128 x 128, k-blocks 32 samples
  const int kb = (n + 31) / 32;
  const int bn = gemm_x3_tile_n(Kin + 1, wide);
  const int tiles = ((Nout + 127) / 128) * ((Kin + bn) / bn);
  DVT_REQUIRE(tiles <= FIT_SEM_TILES, "fit: %d weight-gradient tiles exceed the split-K counters", tiles);
  int splits = std::max(1, std::min(std::min(num_sms(), sm_cap) / std::max(tiles, 1), kb / 4));
  GemmShape s{Nout, Kin + 1, n, splits};
  s.a_mn = 1; s.b_mn = 1; s.x3 = x3; s.plane_a = dY.plane; s.plane_b = X.plane; s.pdl = pdl; s.prio_drop = prio_drop;
  s.x3_wide_min_n = wide;
  return launch_gemm_tn(dY.p, dY.ld, X.p, X.ld, TMAP_F32, s, e, st, impl);
}

// Sweep launch geometry: n > 0 persistent CTAs of 1024 threads (one per SM: the register file is full, so the GEMM
// chain of the next steps keeps the other SMs), else 8 x #SM CTAs of 256 threads (fastest when running alone).
static void fit_sweep_geometry(const Fit* f, bool phase2, int* grid, int* block) {
  const int ctas = f->sweep_ctas[phase2 ? 1 : 0];
  if (ctas > 0) { *grid = ctas; *block = f->sweep_threads; }
  else { *grid = num_sms() * 8; *block = 256; }
}

static int fit_launch_sweep_tma(Fit* f, int ctas, int step_off, int buf_off, cudaStream_t st, bool pdl) {
  static bool prepared = false;
  if (!prepared) {
    DVT_CUDA_OK(cudaFuncSetAttribute(fit_adam_table_tma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SW_SMEM));
    prepared = true;
  }
  DVT_CUDA_OK(launch_k(pdl, fit_adam_table_tma_kernel, dim3(ctas), dim3(SW_THREADS), SW_SMEM, st, f->tb,
                       (uint32_t)(f->n_table / FIT_F), f->sc_main, f->step_base, step_off, buf_off, f->wd));
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// The sweep kernel instance with a window capacity KW >= len (the smallest one: registers).
static int fit_launch_sweep_kernel(Fit* f, dim3 grid, dim3 block, int step_off, int len, int buf_off, cudaStream_t st,
                                   bool pdl) {
  auto go = [&](auto kern) {
    return launch_k(pdl, kern, grid, block, 0, st, f->tb, f->n_table / 4, f->sc_main, f->step_base, step_off, len, buf_off,
                    f->wd);
  };
  static_assert(FIT_MAX_WINDOW <= 8, "add a sweep kernel instance");
  DVT_REQUIRE(len >= 1 && len <= FIT_MAX_WINDOW, "fit: sweep window of %d steps", len);
  if (len == 1) DVT_CUDA_OK(go(fit_adam_table_kernel<1>));
  else if (len <= 2) DVT_CUDA_OK(go(fit_adam_table_kernel<2>));
  else if (len <= 4) DVT_CUDA_OK(go(fit_adam_table_kernel<4>));
  else DVT_CUDA_OK(go(fit_adam_table_kernel<8>));
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// Sweep of the window [step_off, step_off + len) from state buffer (step_base[1] + buf_off) & 1.
static int fit_launch_sweep(Fit* f, int step_off, int len, int buf_off, bool phase2, cudaStream_t st) {
  const bool pdl = f->pdl && f->sweep_pdl;
  if (f->sweep_tma && f->sweep_ctas[phase2 ? 1 : 0] > 0 && len == 1)
    return fit_launch_sweep_tma(f, f->sweep_ctas[phase2 ? 1 : 0], step_off, buf_off, st, pdl);
  int sg_ = 0, sb_ = 0;
  fit_sweep_geometry(f, phase2, &sg_, &sb_);
  return fit_launch_sweep_kernel(f, dim3(sg_), dim3(sb_), step_off, len, buf_off, st, pdl);
}

// Encodes step (*step_base + step_off) into f->enc from state S_{step - npeek} in buffer (step_base[1] + buf_off) & 1,
// applying the npeek pending Adam steps on the fly.
static int fit_enqueue_encode(Fit* f, int step_off, int npeek, int buf_off, cudaStream_t st) {
  const int n = f->bsz;
  const StepRows sr{nullptr, f->step_base, step_off, f->inputs_dev};
  const int tb = 256, blocks = (n * f->grid.n_levels * 4 + tb - 1) / tb;
  auto go = [&](auto kern) {
    return launch_k(f->pdl, kern, dim3(blocks), dim3(tb), 0, st, f->grid, f->tb, nullptr, f->coords, sr, n, f->enc, f->ld_enc,
                    (size_t)n * f->ld_enc, f->sc_main, f->wd, npeek, buf_off);
  };
  static_assert(2 * FIT_MAX_WINDOW <= 16, "add an encode kernel instance");
  DVT_REQUIRE(npeek >= 0 && npeek <= 2 * FIT_MAX_WINDOW, "fit: encode with %d pending steps", npeek);
  if (npeek <= 2) DVT_CUDA_OK(go(fit_encode_kernel<2>));
  else if (npeek <= 4) DVT_CUDA_OK(go(fit_encode_kernel<4>));
  else if (npeek <= 8) DVT_CUDA_OK(go(fit_encode_kernel<8>));
  else if (npeek <= 10) DVT_CUDA_OK(go(fit_encode_kernel<10>));
  else DVT_CUDA_OK(go(fit_encode_kernel<16>));
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  return DVT_OK;
}

// One optimisation step.  epoch_end: the last step before the sweeps are joined (end of a graph, or a plain step).
// Pipelined schedule (f->pipe[phase]): the dense table sweep -- half of a step's time when run in line -- is taken off the
// critical path entirely, and makes one pass over the table per window of up to k = f->sweep_steps[phase] steps.  The
// steps of an epoch form windows [b_0, b_1), [b_1, b_2), ... of k steps (the last one shorter when the epoch ends
// first).  Sweep(w) runs on stream sD, on its own SMs, beside the chains of windows w+1 and w+2:
//   main stream : GEMM h1, GEMM F, [join residual fwd], loss, dgrad, dgrad, [first step of window w: wait sweep(w-2)],
//                 grid backward, [join side chains], encode(t+1) from S_{b_{w-1}} (S_{b_0} in window 0) with Adam steps
//                 b_{w-1} .. t applied on the fly, [last step of window w: fork sweep(w)]
//   side B / C  : weight-gradient GEMMs, residual MLP forward / backward, Adam(small params)
//   side D      : sweep(w): S_{b_w} + g_{b_w} .. g_{b_{w+1}-1} -> S_{b_{w+1}} (the other state buffer)
// The on-the-fly updates use the same adam1() arithmetic on the same inputs as the sweep, so the encoded values are
// bit-identical to a sequential schedule.  Hazards: the encodes of window w read S_{b_{w-1}}, complete since sweep(w-2)
// was waited for, and the gradients of windows w-1 and w; sweep(w) overwrites the buffer of S_{b_{w-1}} and is forked
// after the last of those encodes; the backward of step t overwrites the gradient ring slot of step t - 2k, which lies
// before window w-1 (see fit_create).  With k = 1 this is the two-step-deep pipeline: one sweep per step, encodes with
// two pending steps.  Precondition: f->enc holds the encoding of step t.
// Sequential schedule (f->pipe[phase] == false): encode(t) at the head of the step, sweep(t) on the main stream at its tail.
static int fit_enqueue_step(Fit* f, int step_off, bool phase2, bool epoch_end, cudaStream_t st, int impl) {
  const int n = f->bsz, C = f->C, H1 = C / 2, Hr = C / 4, Lf = f->Lf;
  const StepRows sr{nullptr, f->step_base, step_off, f->inputs_dev};
  const int tb = 256;
  const int enc_blocks = (n * f->grid.n_levels + tb - 1) / tb;
  float* sp = f->sp; float* sg = f->sg;
  const size_t wp = (size_t)f->n_small;  // weight plane stride
  auto W = [&](const Seg& sgm) { return Op{f->wsplit + sgm.off, sgm.cols, wp}; };
  const size_t p_enc = (size_t)n * f->ld_enc, p_h1 = (size_t)n * f->ld_h1, p_nc = (size_t)n * C, p_nh = (size_t)n * H1;
  const size_t p_raw = (size_t)n * f->ld_raw, p_r = (size_t)n * f->ld_r, p_nr = (size_t)n * Hr;
  const Op enc{f->enc, f->ld_enc, p_enc}, h1{f->h1, f->ld_h1, p_h1}, dpred{f->dpred, C, p_nc}, dh1{f->dh1, H1, p_nh};
  const Op rawb{f->rawb, f->ld_raw, p_raw}, r1{f->r1, f->ld_r, p_r}, r2{f->r2, f->ld_r, p_r};
  const Op dR{f->dR, C, p_nc}, dr2{f->dr2, Hr, p_nr}, dr1{f->dr1, Hr, p_nr};
  cudaStream_t sB = f->sB, sC = f->sC, sD = f->sD, sE = f->sE;
  const bool pdl = f->pdl;
  // Kernels that only feed Adam(small) -- weight gradients, the residual MLP's backward, the dG scatter -- can be launched
  // below the chain's priority (DVT_FIT_OFFPATH_PRIO; measured neutral, see fit_create).  What does help is keeping the
  // weight-gradient GEMMs small (wcap): the CUPTI timeline (tools/fit_timeline.py) shows the next kernel of the critical
  // path waiting one CTA lifetime (~12 us, twice per step) whenever a finishing data-gradient GEMM hands its SMs to the
  // queued CTAs of a weight-gradient GEMM -- every 3xTF32 CTA fills the shared memory of its SM.
  const int off = f->off_path_prio_drop;
  const int wide = f->x3_wide_min_n[phase2 ? 1 : 0], wcap = f->wgrad_sms;
  auto fork = [&](cudaStream_t to, cudaEvent_t e) -> int {
    DVT_CUDA_OK(cudaEventRecord(e, st));
    DVT_CUDA_OK(cudaStreamWaitEvent(to, e, 0));
    return DVT_OK;
  };
  auto join = [&](cudaStream_t from, cudaEvent_t e) -> int {
    DVT_CUDA_OK(cudaEventRecord(e, from));
    DVT_CUDA_OK(cudaStreamWaitEvent(st, e, 0));
    return DVT_OK;
  };
  // ---- forward ----
  FIT_RC(fork(sB, f->ev[0]));  // side B: gather the sampled bank rows (+ residual MLP forward in phase 2)
  DVT_CUDA_OK(launch_k(pdl, fit_gather_rows_kernel, dim3(n), dim3(192), 0, sB, f->bank, C, sr, n, f->rawb, f->ld_raw, p_raw));
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  const bool pipe = f->pipe[phase2 ? 1 : 0];
  if (!pipe) FIT_RC(fit_enqueue_encode(f, step_off, 0, f->epoch_windows, st));  // else f->enc is already this step's (fit_run)
  if (phase2) {
    FIT_RC(fit_linear(rawb, n, C, W(f->R1), Hr, sp + f->rb1.off, ACT_RELU, f->r1, f->ld_r, p_r, true, sB, impl, pdl, f->res_x3, 0, wide));
    FIT_RC(fit_linear(r1, n, Hr, W(f->R2), Hr, sp + f->rb2.off, ACT_RELU, f->r2, f->ld_r, p_r, true, sB, impl, pdl, f->res_x3, 0, wide));
    FIT_RC(fit_linear(r2, n, Hr, W(f->R3), C, sp + f->rb3.off, ACT_NONE, f->Rout, C, 0, false, sB, impl, pdl, f->res_x3, 0, wide));
  }
  FIT_RC(fit_linear(enc, n, Lf, W(f->W1), H1, sp + f->b1.off, ACT_RELU, f->h1, f->ld_h1, p_h1, true, st, impl, pdl, 1, 0, wide));
  FIT_RC(fit_linear(h1, n, H1, W(f->W2), C, sp + f->b2.off, ACT_NONE, f->Fout, C, 0, false, st, impl, pdl, 1, 0, wide));
  FIT_RC(join(sB, f->ev[1]));
  // ---- loss + d pred ----
  LossArgs la;
  la.raw = f->rawb; la.ld_raw = f->ld_raw; la.raw_plane = p_raw; la.sr = sr; la.F = f->Fout; la.G = sp + f->G.off; la.R = phase2 ? f->Rout : nullptr;
  la.dpred = f->dpred; la.dR = phase2 ? f->dR : nullptr; la.plane = p_nc;
  la.gG = nullptr;  // dG is scattered by fit_g_scatter_kernel on side C (phase 1), off the critical path
  la.losses = f->losses; la.n = n; la.C = C; la.hw = f->hw; la.loss_scale = f->loss_scale;
  la.ax_i0 = f->ax_i0; la.ax_w0 = f->ax_w0; la.ax_w1 = f->ax_w1; la.gw = f->gw; la.gh = f->gh;
  FIT_RC(launch_loss(la, st, pdl));
  // ---- backward ----
  FIT_RC(fork(sB, f->ev[2]));
  if (phase2) {
    FIT_RC(fork(sC, f->ev[3]));
    FIT_RC(fork(sE, f->ev[11]));
  }
  FIT_RC(fit_wgrad(dpred, n, C, h1, H1, sg + f->W2.off, sg + f->b2.off, f->wg_sem + 0 * FIT_SEM_TILES, sB, impl, pdl, f->wgrad_x3, off, wide, wcap));   // side B
  FIT_RC(fit_dgrad(dpred, n, C, W(f->W2), H1, f->h1, f->ld_h1, f->dh1, H1, p_nh, true, st, impl, pdl, 1, 0, wide));  // main
  FIT_RC(fork(sB, f->ev[4]));  // dh1 ready
  FIT_RC(fit_wgrad(dh1, n, H1, enc, Lf, sg + f->W1.off, sg + f->b1.off, f->wg_sem + 1 * FIT_SEM_TILES, sB, impl, pdl, f->wgrad_x3, off, wide, wcap));  // side B (reads enc)
  FIT_RC(fit_dgrad(dh1, n, H1, W(f->W1), Lf, nullptr, 0, f->denc, Lf, 0, false, st, impl, pdl, 1, 0, wide));
  if (!phase2) {
    // dG (+ grid_sample's neighbour shares) on side C, enqueued BEHIND the two data-gradient GEMMs: launched beside them, its
    // 256 small CTAs take the registers the GEMM CTAs need and delay the critical path.
    FIT_RC(fork(sC, f->ev[3]));
    ScatterArgs sa;
    sa.dpred = f->dpred; sa.plane = p_nc; sa.sr = sr; sa.gG = sg + f->G.off; sa.n = n; sa.C = C; sa.hw = f->hw;
    sa.gw = f->gw; sa.gh = f->gh; sa.ax_i0 = f->ax_i0; sa.ax_w0 = f->ax_w0; sa.ax_w1 = f->ax_w1;
    DVT_CUDA_OK(launch_kx(LaunchOpt{pdl, off}, fit_g_scatter_kernel, dim3((f->hw * 32 + tb - 1) / tb), dim3(tb), 0, sC, sa));
    DVT_CUDA_OK(cudaGetLastError());
    count_launch();
  }
  // the first backward of window w waits for sweep(w-2): the last reader of the gradient slots this window overwrites,
  // and the producer of the state the encodes of this window read
  const int w = f->epoch_windows, j = f->epoch_steps - f->win_first;  // window of this step, position in it
  if (pipe && j == 0 && w >= 2) DVT_CUDA_OK(cudaStreamWaitEvent(st, f->ev_sweep[(w - 2) % 3], 0));
  DVT_CUDA_OK(launch_k(pdl, fit_grid_bwd_kernel, dim3(f->grid.n_levels, GB_PARTS), dim3(GB_THREADS), (size_t)GB_SMEM, st, f->grid,
                       f->coords, sr, n, f->denc, Lf, f->tb));
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  if (phase2) {
    // residual MLP backward: the data-gradient chain on side C, the weight-gradient GEMMs that do not feed it on side E
    //   side C: dr2 = dR.R3 -> dr1 = dr2.R2 -> dR1      side E: dR3 (needs dR, r2 only) -> [dr2 ready] dR2
    FIT_RC(fit_dgrad(dR, n, C, W(f->R3), Hr, f->r2, f->ld_r, f->dr2, Hr, p_nr, true, sC, impl, pdl, f->res_x3, off, wide));
    DVT_CUDA_OK(cudaEventRecord(f->ev[12], sC));                                              // dr2 ready
    FIT_RC(fit_dgrad(dr2, n, Hr, W(f->R2), Hr, f->r1, f->ld_r, f->dr1, Hr, p_nr, true, sC, impl, pdl, f->res_x3, off, wide));
    FIT_RC(fit_wgrad(dr1, n, Hr, rawb, C, sg + f->R1.off, sg + f->rb1.off, f->wg_sem + 2 * FIT_SEM_TILES, sC, impl, pdl, f->res_x3, off, wide, wcap));
    FIT_RC(fit_wgrad(dR, n, C, r2, Hr, sg + f->R3.off, sg + f->rb3.off, f->wg_sem + 3 * FIT_SEM_TILES, sE, impl, pdl, f->res_x3, off, wide, wcap));
    DVT_CUDA_OK(cudaStreamWaitEvent(sE, f->ev[12], 0));
    FIT_RC(fit_wgrad(dr2, n, Hr, r1, Hr, sg + f->R2.off, sg + f->rb2.off, f->wg_sem + 4 * FIT_SEM_TILES, sE, impl, pdl, f->res_x3, off, wide, wcap));
    FIT_RC(join(sE, f->ev[13]));
  }
  FIT_RC(join(sC, f->ev[5]));
  FIT_RC(join(sB, f->ev[6]));  // all small-parameter gradients complete; enc no longer read by a wgrad
  // ---- Adam(small) on side B, beside the table work ----
  FIT_RC(fork(sB, f->ev[7]));
  const int nv = f->n_small / 4;
  DVT_CUDA_OK(launch_k(pdl, fit_adam_small_kernel, dim3((nv + 255) / 256), dim3(256), 0, sB, (float4*)f->sp, (float4*)f->sm,
                       (float4*)f->sv, (float4*)f->sg, f->wsplit, nv, f->G.off / 4,
                       (f->G.off + r8(f->G.rows * f->G.cols)) / 4, f->R1.off / 4, f->n_small / 4, f->sc_main, f->sc_res,
                       f->step_base, step_off, f->freeze_step, f->wd));
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  if (!pipe) {
    FIT_RC(fit_launch_sweep(f, step_off, 1, f->epoch_windows, phase2, st));
    FIT_RC(join(sB, f->ev[8]));
    f->epoch_steps += 1;
    f->epoch_windows += 1;
    f->enc_ready = false;
    return DVT_OK;
  }
  // ---- encode of the NEXT step, from the state before the previous window (the epoch's first state in window 0) ----
  const int read_first = w >= 1 ? f->prev_first : 0;
  FIT_RC(fit_enqueue_encode(f, step_off + 1, f->epoch_steps + 1 - read_first, std::max(w - 1, 0), st));
  FIT_RC(join(sB, f->ev[8]));
  // ---- dense table sweep of the window this step closes ----
  if (j + 1 == f->sweep_steps[phase2 ? 1 : 0] || epoch_end) {
    FIT_RC(fork(sD, f->ev[10]));
    FIT_RC(fit_launch_sweep(f, step_off - j, j + 1, w, phase2, sD));
    DVT_CUDA_OK(cudaEventRecord(f->ev_sweep[w % 3], sD));
    f->epoch_forked = true;
    f->epoch_windows += 1;
    f->prev_first = f->win_first;
    f->win_first = f->epoch_steps + 1;
  }
  f->epoch_steps += 1;
  f->enc_ready = true;
  return DVT_OK;
}

// Waits (on `st`) for all pending table sweeps (sD executes them in order: the last event covers the others) and starts
// a new epoch.  Returns the number of sweeps the epoch enqueued.
static int fit_sync_sweep(Fit* f, cudaStream_t st, int* sweeps) {
  if (f->epoch_forked) {
    DVT_REQUIRE(f->win_first == f->epoch_steps, "fit: an epoch ends inside a sweep window");
    DVT_CUDA_OK(cudaStreamWaitEvent(st, f->ev_sweep[(f->epoch_windows - 1) % 3], 0));
  }
  *sweeps = f->epoch_windows;
  f->epoch_steps = f->epoch_windows = f->win_first = f->prev_first = 0;
  f->epoch_forked = false;
  return DVT_OK;
}

static int fit_capture(Fit* f, bool phase2, int steps, cudaStream_t st, int impl, cudaGraphExec_t* out, long long* nodes,
                       int* sweeps) {
  cudaGraph_t graph = nullptr;
  const long long before = launch_count();
  DVT_CUDA_OK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  int rc = DVT_OK;
  // graphs start and end with the sweeps joined
  f->epoch_steps = f->epoch_windows = f->win_first = f->prev_first = 0;
  f->epoch_forked = false;
  for (int i = 0; i < steps && rc == DVT_OK; ++i) rc = fit_enqueue_step(f, i, phase2, i + 1 == steps, st, impl);
  if (rc == DVT_OK) rc = fit_sync_sweep(f, st, sweeps);  // a capture must join every forked stream
  if (rc == DVT_OK) {
    fit_advance_kernel<<<1, 1, 0, st>>>(f->step_base, steps, *sweeps);
    if (cudaGetLastError() != cudaSuccess) rc = DVT_ERR_CUDA;
    count_launch();
  }
  *nodes = launch_count() - before;
  count_launch(-*nodes);  // captured, not executed
  cudaError_t e = cudaStreamEndCapture(st, &graph);
  if (rc != DVT_OK) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  DVT_CUDA_OK(e);
  if (getenv("DVT_FIT_DEBUG_GRAPH")) {  // what the capture recorded: kernel nodes per priority, programmatic edges
    size_t nn = 0, ne = 0;
    cudaGraphGetNodes(graph, nullptr, &nn);
    std::vector<cudaGraphNode_t> nodes_v(nn);
    cudaGraphGetNodes(graph, nodes_v.data(), &nn);
    int hist[16] = {}, kernels = 0;
    for (auto nd : nodes_v) {
      cudaGraphNodeType ty;
      if (cudaGraphNodeGetType(nd, &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel) continue;
      cudaLaunchAttributeValue v = {};
      if (cudaGraphKernelNodeGetAttribute(nd, cudaLaunchAttributePriority, &v) == cudaSuccess) hist[std::min(15, std::abs(v.priority))] += 1;
      ++kernels;
    }
    cudaGraphGetEdges_v2(graph, nullptr, nullptr, nullptr, &ne);
    std::vector<cudaGraphNode_t> from(ne), to(ne);
    std::vector<cudaGraphEdgeData> ed(ne);
    int prog = 0;
    if (cudaGraphGetEdges_v2(graph, from.data(), to.data(), ed.data(), &ne) == cudaSuccess)
      for (auto& d : ed) prog += d.type == cudaGraphDependencyTypeProgrammatic;
    fprintf(stderr, "[dvt fit graph] phase %d: %zu nodes, %d kernels, |priority| histogram:", phase2 ? 2 : 1, nn, kernels);
    for (int i = 0; i < 16; ++i) if (hist[i]) fprintf(stderr, " %d:%d", i, hist[i]);
    fprintf(stderr, "; %zu edges, %d programmatic\n", ne, prog);
    cudaGetLastError();
  }
  e = cudaGraphInstantiate(out, graph, 0);
  cudaGraphDestroy(graph);
  DVT_CUDA_OK(e);
  return DVT_OK;
}

// Runs steps [cur, cur + count) of the schedule installed by fit_begin.  use_graphs: 0 = plain launches,
// k > 0 = CUDA graphs of k steps each (remainders and the phase boundary fall back to plain launches).
int fit_run(Fit* f, int count, int use_graphs, cudaStream_t caller, int impl) {
  DVT_REQUIRE(f->bank && f->idx[0], "fit_run: call fit_begin first");
  int cur = f->cur_step;  // host mirror of the device step counter: no read-back, no host synchronisation
  // order the engine's stream after everything already enqueued on the caller's stream (the bank is produced there)
  cudaStream_t st = f->stream;
  FIT_RC(fit_after_caller(f, caller));
  DVT_REQUIRE(count >= 0 && cur + count <= f->num_iters, "fit_run: %d steps from %d exceed the schedule of %d", count, cur,
              f->num_iters);
  const int end = cur + count;
  if (use_graphs > 0 && use_graphs != f->graph_steps) {
    fit_drop_graphs(f);
    f->graph_steps = use_graphs;
  }
  while (cur < end) {
    const bool phase2 = cur > f->freeze_step;
    // last step (exclusive) of the current phase within [cur, end)
    const int phase_end = phase2 ? end : std::min(end, f->freeze_step + 1);
    if (f->pipe[phase2 ? 1 : 0] && !f->enc_ready) {
      // a pipelined step expects its encoding in f->enc (first step of a fit / after a sequential step): plain encode,
      // all sweeps are joined here
      FIT_RC(fit_enqueue_encode(f, 0, 0, 0, st));
      f->enc_ready = true;
    }
    if (use_graphs > 0 && cur + use_graphs <= phase_end) {
      cudaGraphExec_t* g = phase2 ? &f->graph2 : &f->graph1;
      long long* nodes = phase2 ? &f->graph2_nodes : &f->graph1_nodes;
      int* sweeps = phase2 ? &f->graph2_sweeps : &f->graph1_sweeps;
      if (!*g) FIT_RC(fit_capture(f, phase2, use_graphs, st, impl, g, nodes, sweeps));
      DVT_CUDA_OK(cudaGraphLaunch(*g, st));
      count_launch(*nodes);
      f->cur_buf ^= *sweeps & 1;
      f->enc_ready = f->pipe[phase2 ? 1 : 0];  // what the captured steps leave behind
      cur += use_graphs;
    } else {
      FIT_RC(fit_enqueue_step(f, 0, phase2, true, st, impl));
      // the sweep reads the device step counter: it must finish before the counter advances
      int sweeps = 0;
      FIT_RC(fit_sync_sweep(f, st, &sweeps));
      fit_advance_kernel<<<1, 1, 0, st>>>(f->step_base, 1, sweeps);
      f->cur_buf ^= sweeps & 1;
      DVT_CUDA_OK(cudaGetLastError());
      count_launch();
      cur += 1;
    }
  }
  f->cur_host = end;
  f->cur_step = end;
  DVT_CUDA_OK(cudaEventRecord(f->ev_run_done[f->idx_slot], st));
  f->run_done_valid[f->idx_slot] = true;
  return fit_before_caller(f, caller);
}

// One dense table sweep (the Adam step of the CURRENT device step counter, state buffer ping-pong not advanced) on `st`:
// the hook bench.py / ncu use to time the dominant HBM-bound kernel alone.  ctas: > 0 persistent 1024-thread CTAs, 0 the
// many-small-CTA geometry.  The optimiser state is modified: call it after the fit results have been read.
int fit_sweep_once(Fit* f, int ctas, cudaStream_t st) {
  DVT_REQUIRE(f->sc_main && f->num_iters > 0, "fit_sweep_once: call fit_begin first");
  // (no device read-back here: a blocking copy per call would put ~20 us of host latency between back-to-back launches
  //  and into every event-timed measurement; the host mirror of the step counter is enough for the bounds check)
  DVT_REQUIRE(f->cur_host <= f->num_iters, "fit_sweep_once: step counter %d beyond the schedule", f->cur_host);
  // ctas > 0: persistent CTAs as in the pipelined schedule (TMA-staged kernel unless DVT_FIT_SWEEP_TMA=0);
  // ctas < 0: -ctas persistent CTAs of the plain-load kernel; 0: the many-small-CTA geometry of the sequential schedule
  if (ctas > 0 && f->sweep_tma) return fit_launch_sweep_tma(f, std::min(ctas, num_sms()), 0, 0, st, false);
  const int n = ctas < 0 ? -ctas : ctas;
  const int grid = n > 0 ? std::min(n, num_sms()) : num_sms() * 8, block = n > 0 ? 1024 : 256;
  return fit_launch_sweep_kernel(f, dim3(grid), dim3(block), 0, 1, 0, st, false);
}

int fit_losses(Fit* f, float* dst_host, int num_iters) {
  DVT_REQUIRE(num_iters == f->num_iters, "fit_losses: schedule has %d steps", f->num_iters);
  DVT_CUDA_OK(cudaStreamSynchronize(f->stream));
  DVT_CUDA_OK(cudaMemcpy(dst_host, f->losses, (size_t)num_iters * 5 * 4, cudaMemcpyDeviceToHost));
  return DVT_OK;
}

// Same table, copied asynchronously on `caller` (dst should be pinned host memory or device memory); the next fit_begin
// is ordered after the copy.
int fit_losses_async(Fit* f, float* dst, int num_iters, cudaStream_t caller) {
  DVT_REQUIRE(num_iters == f->num_iters, "fit_losses: schedule has %d steps", f->num_iters);
  FIT_RC(fit_before_caller(f, caller));
  DVT_CUDA_OK(cudaMemcpyAsync(dst, f->losses, (size_t)num_iters * 5 * 4, cudaMemcpyDefault, caller));
  return DVT_OK;
}

static int fit_query_reserve(Fit* f, int n) {
  if (n <= f->q_cap) return DVT_OK;
  cudaFree(f->q_enc); cudaFree(f->q_h1); cudaFree(f->q_raw); cudaFree(f->q_r1); cudaFree(f->q_r2);
  f->q_enc = f->q_h1 = f->q_raw = f->q_r1 = f->q_r2 = nullptr; f->q_cap = 0;
  DVT_CUDA_OK(cudaMalloc(&f->q_enc, (size_t)n * f->ld_enc * 8));
  DVT_CUDA_OK(cudaMalloc(&f->q_h1, (size_t)n * f->ld_h1 * 8));
  DVT_CUDA_OK(cudaMalloc(&f->q_raw, (size_t)n * f->ld_raw * 8));
  DVT_CUDA_OK(cudaMalloc(&f->q_r1, (size_t)n * f->ld_r * 8));
  DVT_CUDA_OK(cudaMalloc(&f->q_r2, (size_t)n * f->ld_r * 8));
  f->q_cap = n;
  return DVT_OK;
}

// denoised_feats = field(coords): NeuralFeatureField.forward on n points (final query, main_img_denoising.py:121-130)
int fit_query(Fit* f, const float* coords, int n, float* out, cudaStream_t st, int impl) {
  DVT_REQUIRE(coords && out && n > 0, "fit_query: bad arguments");
  FIT_RC(fit_query_reserve(f, n));
  FIT_RC(fit_before_caller(f, st));
  const int C = f->C, H1 = C / 2;
  const size_t cap = (size_t)f->q_cap, wp = (size_t)f->n_small;
  const StepRows sr{nullptr, f->step_base, 0};
  fit_encode_kernel<2><<<(n * f->grid.n_levels * 4 + 255) / 256, 256, 0, st>>>(
      f->grid, f->tb, f->tb.p[f->cur_buf], coords, sr, n, f->q_enc, f->ld_enc, cap * f->ld_enc, nullptr, 0.f, 0, 0);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  FIT_RC(fit_linear(Op{f->q_enc, f->ld_enc, cap * f->ld_enc}, n, f->Lf, Op{f->wsplit + f->W1.off, f->Lf, wp}, H1,
                    f->sp + f->b1.off, ACT_RELU, f->q_h1, f->ld_h1, cap * f->ld_h1, true, st, impl));
  FIT_RC(fit_linear(Op{f->q_h1, f->ld_h1, cap * f->ld_h1}, n, H1, Op{f->wsplit + f->W2.off, H1, wp}, C, f->sp + f->b2.off,
                    ACT_NONE, out, C, 0, false, st, impl));
  return DVT_OK;
}

// pred_residual = residual_predictor(raw) on n rows (offline_denoiser.py:40-46,105)
int fit_residual(Fit* f, const float* raw, int n, float* out, cudaStream_t st, int impl) {
  DVT_REQUIRE(raw && out && n > 0, "fit_residual: bad arguments");
  FIT_RC(fit_query_reserve(f, n));
  FIT_RC(fit_before_caller(f, st));
  const int C = f->C, Hr = C / 4;
  const size_t cap = (size_t)f->q_cap, wp = (size_t)f->n_small;
  const StepRows sr{nullptr, f->step_base, 0};
  fit_gather_rows_kernel<<<n, 192, 0, st>>>(raw, C, sr, n, f->q_raw, f->ld_raw, cap * f->ld_raw);
  DVT_CUDA_OK(cudaGetLastError());
  count_launch();
  FIT_RC(fit_linear(Op{f->q_raw, f->ld_raw, cap * f->ld_raw}, n, C, Op{f->wsplit + f->R1.off, C, wp}, Hr, f->sp + f->rb1.off,
                    ACT_RELU, f->q_r1, f->ld_r, cap * f->ld_r, true, st, impl));
  FIT_RC(fit_linear(Op{f->q_r1, f->ld_r, cap * f->ld_r}, n, Hr, Op{f->wsplit + f->R2.off, Hr, wp}, Hr, f->sp + f->rb2.off,
                    ACT_RELU, f->q_r2, f->ld_r, cap * f->ld_r, true, st, impl));
  FIT_RC(fit_linear(Op{f->q_r2, f->ld_r, cap * f->ld_r}, n, Hr, Op{f->wsplit + f->R3.off, Hr, wp}, C, f->sp + f->rb3.off,
                    ACT_NONE, out, C, 0, false, st, impl));
  return DVT_OK;
}

// unit-test entry points ---------------------------------------------------------------------------------
static int levels_from_arrays(GridLevels* g, int n_levels, const float* scale, const uint32_t* res, const uint32_t* size,
                              const uint32_t* offset, const uint32_t* hashed) {
  DVT_REQUIRE(n_levels >= 1 && n_levels <= FIT_MAX_LEVELS, "hashgrid: n_levels %d out of range", n_levels);
  g->n_levels = n_levels;
  for (int l = 0; l < n_levels; ++l) {
    g->scale[l] = scale[l]; g->res[l] = res[l]; g->size[l] = size[l]; g->offset[l] = offset[l]; g->hashed[l] = hashed[l];
  }
  g->offset[n_levels] = offset[n_levels];
  return DVT_OK;
}

int hashgrid_corners(int n_levels, const float* scale, const uint32_t* res, const uint32_t* size, const uint32_t* offset,
                     const uint32_t* hashed, const float* coords, int n, uint32_t* idx, float* w, cudaStream_t st) {
  GridLevels g;
  FIT_RC(levels_from_arrays(&g, n_levels, scale, res, size, offset, hashed));
  fit_corners_kernel<<<(n * n_levels + 255) / 256, 256, 0, st>>>(g, coords, n, idx, w);
  DVT_CUDA_OK(cudaGetLastError());
  return DVT_OK;
}

int hashgrid_fwd(int n_levels, const float* scale, const uint32_t* res, const uint32_t* size, const uint32_t* offset,
                 const uint32_t* hashed, const float* table, const float* coords, int n, float* out, cudaStream_t st) {
  GridLevels g;
  FIT_RC(levels_from_arrays(&g, n_levels, scale, res, size, offset, hashed));
  fit_encode_f32_kernel<<<(n * n_levels + 255) / 256, 256, 0, st>>>(g, table, coords, n, out);
  DVT_CUDA_OK(cudaGetLastError());
  return DVT_OK;
}

int hashgrid_bwd(int n_levels, const float* scale, const uint32_t* res, const uint32_t* size, const uint32_t* offset,
                 const uint32_t* hashed, const float* coords, int n, const float* dout, float* gtable, cudaStream_t st) {
  GridLevels g;
  FIT_RC(levels_from_arrays(&g, n_levels, scale, res, size, offset, hashed));
  const StepRows sr{nullptr, nullptr, 0};
  TableBufs tb = {};
  tb.g = gtable;  // no stamps: plain accumulation
  FIT_RC(fit_prepare_kernels());
  fit_grid_bwd_kernel<<<dim3(n_levels, GB_PARTS), GB_THREADS, GB_SMEM, st>>>(g, coords, sr, n, dout, n_levels * FIT_F, tb);
  DVT_CUDA_OK(cudaGetLastError());
  return DVT_OK;
}

int fit_n_small(const Fit* f) { return f->n_small; }
size_t fit_n_table(const Fit* f) { return f->n_table; }

}  // namespace dvt
