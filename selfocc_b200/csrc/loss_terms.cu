// Per-sample regularisers of the training objective (SURVEY.md 8f-2): the mean of an elementwise function over a large
// fp32 tensor and the gradient of that mean.  EikonalLoss (loss/eikonal_loss.py:19-21), SecondGradLoss
// (loss/second_grad_loss.py:19-20) and SoftSparsityLoss (loss/sparsity_loss.py:80-81).
//
// Forward: one read.  A fixed grid (a function of n only, never of the device) strides over 128-bit words; every CTA
// accumulates in fp64 and writes one partial, and a one-CTA launch sums the partials in index order and writes the fp32
// mean.  No float atomics: the result is bitwise repeatable on any device.
// Backward: one read of x and one write of grad_x, the scale grad_out[0] / count read on the device.
//
// The same two launches serve SparsityLoss (sparsity_loss.py:24-27) and HardSparsityLoss (:49-63) on the uniform_sdf
// lattice, and AdaptiveSparsityLoss (:102-114) runs per ray: one warp reduces a ray's masked samples to (sum, count) in
// fp64, and a fixed-grid reduction of those per-ray pairs gives the ratio.
#include <algorithm>
#include <cmath>
#include "eikonal_terms.cuh"

namespace so {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxPartials = SO_SAMPLE_MEAN_WORKSPACE_BYTES / 8;
static_assert(kMaxPartials == 1024, "the finalising CTA reduces one partial per thread");

// internal op codes of the lattice terms (not part of the C ABI's SO_SAMPLE_MEAN_* set)
constexpr int kOpSparsity = 16;
constexpr int kOpHardSparsity = 17;

// parameters of the lattice terms; ABS / NEG_RELU / EIKONAL ignore them
struct TermParams {
  float scale;             // SPARSITY: the loss's scale; HARD: the sigmoid's slope
  float thresh;            // HARD: the relu's threshold
  uint32_t H, W, D;        // HARD: lattice dims, x is [H, W, D]
  uint32_t lo[3], hi[3];   // HARD: cells outside [lo, hi) per axis are cropped (read as 100)
  const float* loss;       // HARD backward: the forward's relu output; the gradient is zero unless it is > 0
};

__device__ __forceinline__ bool cropped(int64_t i, const TermParams& p) {
  const uint32_t u = (uint32_t)i, d = u % p.D, hw = u / p.D, w = hw % p.W, h = hw / p.W;
  return h < p.lo[0] || h >= p.hi[0] || w < p.lo[1] || w >= p.hi[1] || d < p.lo[2] || d >= p.hi[2];
}

// sech^2(u) = 4e / (1 + e)^2 and tanh(|u|) = (1 - e) / (1 + e) with e = exp(-2|u|) <= 1: finite for every finite u and 0
// (not cosh's inf / inf) once e underflows
__device__ __forceinline__ float sech2(float u) {
  const float e = expf(-2.f * fabsf(u)), q = 1.f + e;
  return 4.f * e / (q * q);
}

__device__ __forceinline__ float sigmoid_neg(float x, float scale) { return 1.f / (1.f + expf(-(x * -scale))); }

// ---- the elementwise functions and their torch subgradients (EIKONAL: eikonal_terms.cuh); i is x's flat index
template <int OP>
__device__ __forceinline__ double f_scalar(float x, int64_t i, const TermParams& p) {
  if (OP == SO_SAMPLE_MEAN_ABS) return (double)fabsf(x);
  if (OP == kOpSparsity) return (double)sech2(x / (2.f * p.scale));
  if (OP == kOpHardSparsity) return (double)sigmoid_neg(cropped(i, p) ? 100.f : x, p.scale);
  return x < 0.f ? -(double)x : 0.0;                               // relu(-x)
}

template <int OP>
__device__ __forceinline__ float df_scalar(float x, float s, int64_t i, const TermParams& p) {
  if (OP == SO_SAMPLE_MEAN_ABS) return x > 0.f ? s : (x < 0.f ? -s : 0.f);   // sign(x) * s, 0 at 0
  if (OP == kOpSparsity) {                                                   // -tanh(u) sech^2(u) / scale
    const float u = x / (2.f * p.scale), a = fabsf(u), e = expf(-2.f * a), q = 1.f + e;
    const float th = copysignf(-expm1f(-2.f * a) / q, u);
    return s * (-th * (4.f * e / (q * q)) / p.scale);
  }
  if (OP == kOpHardSparsity) {                                               // -scale sigma (1 - sigma), 0 where cropped
    if (cropped(i, p)) return 0.f;
    const float sg = sigmoid_neg(x, p.scale);
    return s * (sg * (1.f - sg)) * -p.scale;
  }
  return x < 0.f ? -s : 0.f;                                                 // 0 at x = 0
}

// Work split: `head` scalar units before the first aligned word, `nvec` vector items, then the tail.  A unit is one
// element (ABS, NEG_RELU) or one row of 3 (EIKONAL); a vector item is one float4 or, for EIKONAL, 3 float4 = 4 rows.
struct Split {
  int64_t units, head, nvec, tail_begin;
};

template <int OP>
Split make_split(const float* x, int64_t n, bool vec) {
  Split s;
  s.units = OP == SO_SAMPLE_MEAN_EIKONAL ? n / 3 : n;
  constexpr int per = 4;                                           // units per vector item: 4 elements or 4 rows
  s.head = 0;
  const int64_t w = (int64_t)(((uintptr_t)x >> 2) & 3);            // float offset inside a 16-byte word
  if (OP == SO_SAMPLE_MEAN_EIKONAL) {
    while ((w + 3 * s.head) & 3) ++s.head;                         // first row that starts a 16-byte word (< 4 rows)
  } else {
    s.head = (4 - w) & 3;
  }
  if (!vec || s.head > s.units) s.head = s.units;
  s.nvec = (s.units - s.head) / per;
  s.tail_begin = s.head + s.nvec * per;
  return s;
}

__device__ __forceinline__ double block_sum(double v, double* sh) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  v = 0.0;
  if (warp == 0) {
    v = lane < (int)(blockDim.x >> 5) ? sh[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  }
  return v;
}

template <int OP>
__global__ void __launch_bounds__(kThreads) sample_mean_partial_kernel(const float* __restrict__ x, Split sp,
                                                                       double* __restrict__ partials, TermParams p) {
  __shared__ double sh[32];
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  double acc = 0.0;
  if (OP == SO_SAMPLE_MEAN_EIKONAL) {
    const float4* v = reinterpret_cast<const float4*>(x + 3 * sp.head);
    for (int64_t i = tid; i < sp.nvec; i += stride) {
      const float4 a = __ldcs(v + 3 * i), b = __ldcs(v + 3 * i + 1), c = __ldcs(v + 3 * i + 2);
      acc += eik_row(a.x, a.y, a.z) + eik_row(a.w, b.x, b.y) + eik_row(b.z, b.w, c.x) + eik_row(c.y, c.z, c.w);
    }
  } else {
    const float4* v = reinterpret_cast<const float4*>(x + sp.head);
    int64_t i = tid;
    for (; i + stride < sp.nvec; i += 2 * stride) {                 // two independent 128-bit loads in flight
      const float4 a = __ldcs(v + i), b = __ldcs(v + i + stride);
      const int64_t ia = sp.head + 4 * i, ib = sp.head + 4 * (i + stride);
      acc += f_scalar<OP>(a.x, ia, p) + f_scalar<OP>(a.y, ia + 1, p) + f_scalar<OP>(a.z, ia + 2, p) +
             f_scalar<OP>(a.w, ia + 3, p) + f_scalar<OP>(b.x, ib, p) + f_scalar<OP>(b.y, ib + 1, p) +
             f_scalar<OP>(b.z, ib + 2, p) + f_scalar<OP>(b.w, ib + 3, p);
    }
    if (i < sp.nvec) {
      const float4 a = __ldcs(v + i);
      const int64_t ia = sp.head + 4 * i;
      acc += f_scalar<OP>(a.x, ia, p) + f_scalar<OP>(a.y, ia + 1, p) + f_scalar<OP>(a.z, ia + 2, p) +
             f_scalar<OP>(a.w, ia + 3, p);
    }
  }
  // unaligned head and tail, unit by unit
  const int64_t n_tail = sp.units - sp.tail_begin;
  for (int64_t j = tid; j < sp.head + n_tail; j += stride) {
    const int64_t u = j < sp.head ? j : sp.tail_begin + (j - sp.head);
    if (OP == SO_SAMPLE_MEAN_EIKONAL)
      acc += eik_row(x[3 * u], x[3 * u + 1], x[3 * u + 2]);
    else
      acc += f_scalar<OP>(x[u], u, p);
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) partials[blockIdx.x] = acc;
}

// kHinge (HardSparsityLoss): out = relu(mean - thresh) in fp32, as the reference's fp32 mean and subtraction; a NaN mean
// stays NaN, as torch.relu keeps it
template <bool kHinge>
__global__ void __launch_bounds__(kMaxPartials) sample_mean_final_kernel(const double* __restrict__ partials, int n_part,
                                                                         int64_t count, float* __restrict__ out,
                                                                         float thresh) {
  __shared__ double sh[32];
  const double v = block_sum((int)threadIdx.x < n_part ? partials[threadIdx.x] : 0.0, sh);
  if (threadIdx.x == 0) {
    const float m = (float)(v / (double)count);
    if (kHinge) {
      const float h = m - thresh;
      out[0] = h > 0.f || h != h ? h : 0.f;
    } else {
      out[0] = m;
    }
  }
}

template <int OP>
__global__ void __launch_bounds__(kThreads) sample_mean_backward_kernel(const float* __restrict__ x, Split sp,
                                                                        const float* __restrict__ g_out, int64_t count,
                                                                        float* __restrict__ gx, TermParams p) {
  float s = (float)((double)__ldg(g_out) / (double)count);
  if (OP == kOpHardSparsity && !(__ldg(p.loss) > 0.f)) s = 0.f;   // relu inactive (or NaN): torch passes no gradient
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  if (OP == SO_SAMPLE_MEAN_EIKONAL) {
    const float4* v = reinterpret_cast<const float4*>(x + 3 * sp.head);
    float4* o = reinterpret_cast<float4*>(gx + 3 * sp.head);
    for (int64_t i = tid; i < sp.nvec; i += stride) {
      float4 a = __ldcs(v + 3 * i), b = __ldcs(v + 3 * i + 1), c = __ldcs(v + 3 * i + 2);
      const float k0 = eik_coef(a.x, a.y, a.z, s), k1 = eik_coef(a.w, b.x, b.y, s);
      const float k2 = eik_coef(b.z, b.w, c.x, s), k3 = eik_coef(c.y, c.z, c.w, s);
      a = make_float4(a.x * k0, a.y * k0, a.z * k0, a.w * k1);
      b = make_float4(b.x * k1, b.y * k1, b.z * k2, b.w * k2);
      c = make_float4(c.x * k2, c.y * k3, c.z * k3, c.w * k3);
      __stcs(o + 3 * i, a);
      __stcs(o + 3 * i + 1, b);
      __stcs(o + 3 * i + 2, c);
    }
  } else {
    const float4* v = reinterpret_cast<const float4*>(x + sp.head);
    float4* o = reinterpret_cast<float4*>(gx + sp.head);
    for (int64_t i = tid; i < sp.nvec; i += stride) {
      const float4 a = __ldcs(v + i);
      const int64_t ia = sp.head + 4 * i;
      __stcs(o + i, make_float4(df_scalar<OP>(a.x, s, ia, p), df_scalar<OP>(a.y, s, ia + 1, p),
                                df_scalar<OP>(a.z, s, ia + 2, p), df_scalar<OP>(a.w, s, ia + 3, p)));
    }
  }
  const int64_t n_tail = sp.units - sp.tail_begin;
  for (int64_t j = tid; j < sp.head + n_tail; j += stride) {
    const int64_t u = j < sp.head ? j : sp.tail_begin + (j - sp.head);
    if (OP == SO_SAMPLE_MEAN_EIKONAL) {
      const float a = x[3 * u], b = x[3 * u + 1], c = x[3 * u + 2];
      const float k = eik_coef(a, b, c, s);
      gx[3 * u] = a * k;
      gx[3 * u + 1] = b * k;
      gx[3 * u + 2] = c * k;
    } else {
      gx[u] = df_scalar<OP>(x[u], s, u, p);
    }
  }
}

// fixed grid: a function of the work size only, so the partials (and the sum) do not depend on the device
unsigned grid_for(const Split& sp) {
  const int64_t work = sp.nvec > 0 ? sp.nvec : sp.units;
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(kMaxPartials, ceil_div64(work, kThreads)));
}

int validate(const float* x, int64_t n, int32_t op) {
  if (!x || n < 1) return SO_ERR_INVALID_ARG;
  if (op != SO_SAMPLE_MEAN_EIKONAL && op != SO_SAMPLE_MEAN_ABS && op != SO_SAMPLE_MEAN_NEG_RELU) return SO_ERR_INVALID_ARG;
  if (op == SO_SAMPLE_MEAN_EIKONAL && n % 3) return SO_ERR_INVALID_ARG;
  if ((uintptr_t)x & 3) return SO_ERR_INVALID_ARG;
  return SO_OK;
}

template <int OP>
void launch_forward(const float* x, int64_t n, double* ws, float* out, cudaStream_t st, const TermParams& p = {}) {
  const Split sp = make_split<OP>(x, n, true);
  const unsigned grid = grid_for(sp);
  sample_mean_partial_kernel<OP><<<grid, kThreads, 0, st>>>(x, sp, ws, p);
  sample_mean_final_kernel<OP == kOpHardSparsity><<<1, kMaxPartials, 0, st>>>(ws, (int)grid, sp.units, out, p.thresh);
}

template <int OP>
void launch_backward(const float* x, int64_t n, const float* g_out, float* gx, cudaStream_t st, const TermParams& p = {}) {
  // 128-bit words of x and grad_x line up only when both sit at the same offset inside a word
  const bool vec = (((uintptr_t)x ^ (uintptr_t)gx) & 15) == 0;
  const Split sp = make_split<OP>(x, n, vec);
  sample_mean_backward_kernel<OP><<<grid_for(sp), kThreads, 0, st>>>(x, sp, g_out, sp.units, gx, p);
}

// ---- the lattice terms' arguments
int validate_lattice(const float* x, int64_t n, float scale) {
  if (!x || n < 1 || ((uintptr_t)x & 3)) return SO_ERR_INVALID_ARG;
  if (!std::isfinite(scale) || scale == 0.f) return SO_ERR_INVALID_ARG;
  return SO_OK;
}

int hard_params(const float* x, int32_t H, int32_t W, int32_t D, const int32_t* crop, float scale, TermParams& p) {
  if (!x || ((uintptr_t)x & 3) || !std::isfinite(scale)) return SO_ERR_INVALID_ARG;      // any finite slope, 0 included
  if (H < 1 || W < 1 || D < 1 || (int64_t)H * W * D > INT32_MAX) return SO_ERR_INVALID_ARG;
  p.scale = scale;
  p.H = (uint32_t)H, p.W = (uint32_t)W, p.D = (uint32_t)D;
  const int32_t dims[3] = {H, W, D};
  for (int a = 0; a < 3; ++a) {
    const int32_t c0 = crop ? crop[2 * a] : 0, c1 = crop ? crop[2 * a + 1] : 0;
    if (c0 < 0 || c1 < 0) return SO_ERR_INVALID_ARG;
    p.lo[a] = (uint32_t)c0;
    p.hi[a] = (uint32_t)std::max<int64_t>(0, (int64_t)dims[a] - c1);
  }
  return SO_OK;
}

// ---- AdaptiveSparsityLoss: one warp per ray, S samples ray-major; a sample counts where ts > depth + slack (fp32, as the
// reference's mask).  The lanes stride over the samples and fold in a fixed shuffle order: deterministic.
constexpr int kRayWarps = kThreads / 32;

__global__ void __launch_bounds__(kThreads) adaptive_rays_kernel(const float* __restrict__ sdf, const float* __restrict__ ts,
                                                                 const float* __restrict__ depth, int64_t n_rays, int S,
                                                                 float slack, double2* __restrict__ stats) {
  const int64_t r = (int64_t)blockIdx.x * kRayWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n_rays) return;
  const float thr = __ldg(depth + r) + slack;
  const float* sr = sdf + r * S;
  const float* tr = ts + r * S;
  double sum = 0.0;
  int cnt = 0;
  for (int j = lane; j < S; j += 32) {
    const float t = __ldcs(tr + j), d = __ldcs(sr + j);
    if (t > thr) {
      ++cnt;
      if (d < 0.f) sum -= (double)d;                              // relu(-sdf)
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_down_sync(0xffffffffu, sum, o);
    cnt += __shfl_down_sync(0xffffffffu, cnt, o);
  }
  if (lane == 0) stats[r] = make_double2(sum, (double)cnt);
}

// d loss / d sdf = -grad_stats[ray].x where the sample counts and sdf < 0 (relu's 0 at sdf = 0), else 0
__global__ void __launch_bounds__(kThreads) adaptive_backward_kernel(const float* __restrict__ sdf,
                                                                     const float* __restrict__ ts,
                                                                     const float* __restrict__ depth, int64_t n_rays,
                                                                     int S, float slack,
                                                                     const double2* __restrict__ g_stats,
                                                                     float* __restrict__ gx) {
  const int64_t r = (int64_t)blockIdx.x * kRayWarps + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n_rays) return;
  const float thr = __ldg(depth + r) + slack;
  const float g = -(float)g_stats[r].x;
  for (int j = lane; j < S; j += 32) {
    const int64_t i = r * S + j;
    gx[i] = __ldcs(ts + i) > thr && __ldcs(sdf + i) < 0.f ? g : 0.f;
  }
}

// the per-ray (sum, count) pairs in a fixed grid (a function of n_rays only), one pair per CTA in the workspace, then one
// CTA sums the pairs in index order: out = sum / count (0 / 0 = NaN for an empty mask, as torch's mean of nothing)
constexpr int kMaxPairs = SO_SAMPLE_MEAN_WORKSPACE_BYTES / 16;

__global__ void __launch_bounds__(kThreads) ray_pairs_partial_kernel(const double2* __restrict__ stats, int64_t n_rays,
                                                                    double2* __restrict__ partials) {
  __shared__ double sh[32];
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  double s = 0.0, c = 0.0;
  for (int64_t r = tid; r < n_rays; r += stride) {
    const double2 v = stats[r];
    s += v.x;
    c += v.y;
  }
  s = block_sum(s, sh);
  __syncthreads();
  c = block_sum(c, sh);
  if (threadIdx.x == 0) partials[blockIdx.x] = make_double2(s, c);
}

__global__ void __launch_bounds__(kMaxPairs) ray_pairs_final_kernel(const double2* __restrict__ partials, int n_part,
                                                                    float* __restrict__ out, double* __restrict__ total) {
  __shared__ double sh[32];
  const double2 v = (int)threadIdx.x < n_part ? partials[threadIdx.x] : make_double2(0.0, 0.0);
  const double s = block_sum(v.x, sh);
  __syncthreads();
  const double c = block_sum(v.y, sh);
  if (threadIdx.x == 0) {
    out[0] = (float)(s / c);
    if (total) total[0] = s, total[1] = c;
  }
}

int validate_rays(const float* sdf, const float* ts, const float* depth, int64_t n_rays, int32_t S, float slack) {
  if (n_rays < 0 || S < 1 || !std::isfinite(slack)) return SO_ERR_INVALID_ARG;
  if (n_rays > 0 && (!sdf || !ts || !depth || (((uintptr_t)sdf | (uintptr_t)ts | (uintptr_t)depth) & 3)))
    return SO_ERR_INVALID_ARG;
  if (n_rays > INT64_MAX / S) return SO_ERR_INVALID_ARG;
  return SO_OK;
}

}  // namespace
}  // namespace so

using namespace so;

extern "C" int so_sample_mean_forward(const float* x, int64_t n, int32_t op, void* workspace, float* out, void* stream) {
  int rc = validate(x, n, op);
  if (rc) return rc;
  if (!workspace || !out || ((uintptr_t)workspace & 7) || ((uintptr_t)out & 3)) return SO_ERR_INVALID_ARG;
  const cudaStream_t st = (cudaStream_t)stream;
  double* ws = (double*)workspace;
  if (op == SO_SAMPLE_MEAN_EIKONAL) launch_forward<SO_SAMPLE_MEAN_EIKONAL>(x, n, ws, out, st);
  else if (op == SO_SAMPLE_MEAN_ABS) launch_forward<SO_SAMPLE_MEAN_ABS>(x, n, ws, out, st);
  else launch_forward<SO_SAMPLE_MEAN_NEG_RELU>(x, n, ws, out, st);
  note_launch(2);
  return check_launch();
}

extern "C" int so_sample_mean_backward(const float* x, int64_t n, int32_t op, const float* grad_out, float* grad_x,
                                       void* stream) {
  int rc = validate(x, n, op);
  if (rc) return rc;
  if (!grad_out || !grad_x || ((uintptr_t)grad_x & 3)) return SO_ERR_INVALID_ARG;
  const cudaStream_t st = (cudaStream_t)stream;
  if (op == SO_SAMPLE_MEAN_EIKONAL) launch_backward<SO_SAMPLE_MEAN_EIKONAL>(x, n, grad_out, grad_x, st);
  else if (op == SO_SAMPLE_MEAN_ABS) launch_backward<SO_SAMPLE_MEAN_ABS>(x, n, grad_out, grad_x, st);
  else launch_backward<SO_SAMPLE_MEAN_NEG_RELU>(x, n, grad_out, grad_x, st);
  note_launch(1);
  return check_launch();
}

extern "C" int so_sparsity_forward(const float* x, int64_t n, float scale, void* workspace, float* out, void* stream) {
  int rc = validate_lattice(x, n, scale);
  if (rc) return rc;
  if (!workspace || !out || ((uintptr_t)workspace & 7) || ((uintptr_t)out & 3)) return SO_ERR_INVALID_ARG;
  TermParams p{};
  p.scale = scale;
  launch_forward<kOpSparsity>(x, n, (double*)workspace, out, (cudaStream_t)stream, p);
  note_launch(2);
  return check_launch();
}

extern "C" int so_sparsity_backward(const float* x, int64_t n, float scale, const float* grad_out, float* grad_x,
                                    void* stream) {
  int rc = validate_lattice(x, n, scale);
  if (rc) return rc;
  if (!grad_out || !grad_x || ((uintptr_t)grad_x & 3)) return SO_ERR_INVALID_ARG;
  TermParams p{};
  p.scale = scale;
  launch_backward<kOpSparsity>(x, n, grad_out, grad_x, (cudaStream_t)stream, p);
  note_launch(1);
  return check_launch();
}

extern "C" int so_hard_sparsity_forward(const float* x, int32_t H, int32_t W, int32_t D, const int32_t* crop, float scale,
                                        float thresh, void* workspace, float* out, void* stream) {
  TermParams p{};
  int rc = hard_params(x, H, W, D, crop, scale, p);
  if (rc) return rc;
  if (!std::isfinite(thresh) || !workspace || !out || ((uintptr_t)workspace & 7) || ((uintptr_t)out & 3))
    return SO_ERR_INVALID_ARG;
  p.thresh = thresh;
  launch_forward<kOpHardSparsity>(x, (int64_t)H * W * D, (double*)workspace, out, (cudaStream_t)stream, p);
  note_launch(2);
  return check_launch();
}

extern "C" int so_hard_sparsity_backward(const float* x, int32_t H, int32_t W, int32_t D, const int32_t* crop, float scale,
                                         const float* loss, const float* grad_out, float* grad_x, void* stream) {
  TermParams p{};
  int rc = hard_params(x, H, W, D, crop, scale, p);
  if (rc) return rc;
  if (!loss || !grad_out || !grad_x || ((uintptr_t)grad_x & 3)) return SO_ERR_INVALID_ARG;
  p.loss = loss;
  launch_backward<kOpHardSparsity>(x, (int64_t)H * W * D, grad_out, grad_x, (cudaStream_t)stream, p);
  note_launch(1);
  return check_launch();
}

extern "C" int so_adaptive_sparsity_rays(const float* sdf, const float* ts, const float* depth, int64_t n_rays, int32_t S,
                                         float slack, double* ray_stats, void* stream) {
  int rc = validate_rays(sdf, ts, depth, n_rays, S, slack);
  if (rc) return rc;
  if (n_rays == 0) return SO_OK;
  if (!ray_stats || ((uintptr_t)ray_stats & 15)) return SO_ERR_INVALID_ARG;
  adaptive_rays_kernel<<<(unsigned)ceil_div64(n_rays, kRayWarps), kThreads, 0, (cudaStream_t)stream>>>(
      sdf, ts, depth, n_rays, S, slack, (double2*)ray_stats);
  note_launch(1);
  return check_launch();
}

extern "C" int so_adaptive_sparsity_reduce(const double* ray_stats, int64_t n_rays, void* workspace, float* out,
                                           double* total, void* stream) {
  if (!ray_stats || n_rays < 1 || !workspace || !out || ((uintptr_t)ray_stats & 15) || ((uintptr_t)workspace & 15) ||
      ((uintptr_t)out & 3) || ((uintptr_t)total & 7))
    return SO_ERR_INVALID_ARG;
  const unsigned grid = (unsigned)std::max<int64_t>(1, std::min<int64_t>(kMaxPairs, ceil_div64(n_rays, kThreads)));
  const cudaStream_t st = (cudaStream_t)stream;
  ray_pairs_partial_kernel<<<grid, kThreads, 0, st>>>((const double2*)ray_stats, n_rays, (double2*)workspace);
  ray_pairs_final_kernel<<<1, kMaxPairs, 0, st>>>((const double2*)workspace, (int)grid, out, total);
  note_launch(2);
  return check_launch();
}

extern "C" int so_adaptive_sparsity_backward(const float* sdf, const float* ts, const float* depth, int64_t n_rays,
                                             int32_t S, float slack, const double* grad_stats, float* grad_sdf,
                                             void* stream) {
  int rc = validate_rays(sdf, ts, depth, n_rays, S, slack);
  if (rc) return rc;
  if (n_rays == 0) return SO_OK;
  if (!grad_stats || !grad_sdf || ((uintptr_t)grad_stats & 15) || ((uintptr_t)grad_sdf & 3)) return SO_ERR_INVALID_ARG;
  adaptive_backward_kernel<<<(unsigned)ceil_div64(n_rays, kRayWarps), kThreads, 0, (cudaStream_t)stream>>>(
      sdf, ts, depth, n_rays, S, slack, (const double2*)grad_stats, grad_sdf);
  note_launch(1);
  return check_launch();
}
