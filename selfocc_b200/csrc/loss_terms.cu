// Per-sample regularisers of the training objective (SURVEY.md 8f-2): the mean of an elementwise function over a large
// fp32 tensor and the gradient of that mean.  EikonalLoss (loss/eikonal_loss.py:19-21), SecondGradLoss
// (loss/second_grad_loss.py:19-20) and SoftSparsityLoss (loss/sparsity_loss.py:80-81).
//
// Forward: one read.  A fixed grid (a function of n only, never of the device) strides over 128-bit words; every CTA
// accumulates in fp64 and writes one partial, and a one-CTA launch sums the partials in index order and writes the fp32
// mean.  No float atomics: the result is bitwise repeatable on any device.
// Backward: one read of x and one write of grad_x, the scale grad_out[0] / count read on the device.
#include <algorithm>
#include "eikonal_terms.cuh"

namespace so {
namespace {

constexpr int kThreads = 256;
constexpr int kMaxPartials = SO_SAMPLE_MEAN_WORKSPACE_BYTES / 8;
static_assert(kMaxPartials == 1024, "the finalising CTA reduces one partial per thread");

// ---- the elementwise functions of ABS and NEG_RELU and their torch subgradients (EIKONAL: eikonal_terms.cuh)
template <int OP>
__device__ __forceinline__ double f_scalar(float x) {
  if (OP == SO_SAMPLE_MEAN_ABS) return (double)fabsf(x);
  return x < 0.f ? -(double)x : 0.0;                               // relu(-x)
}

template <int OP>
__device__ __forceinline__ float df_scalar(float x, float s) {
  if (OP == SO_SAMPLE_MEAN_ABS) return x > 0.f ? s : (x < 0.f ? -s : 0.f);   // sign(x) * s, 0 at 0
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
                                                                       double* __restrict__ partials) {
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
      acc += f_scalar<OP>(a.x) + f_scalar<OP>(a.y) + f_scalar<OP>(a.z) + f_scalar<OP>(a.w) +
             f_scalar<OP>(b.x) + f_scalar<OP>(b.y) + f_scalar<OP>(b.z) + f_scalar<OP>(b.w);
    }
    if (i < sp.nvec) {
      const float4 a = __ldcs(v + i);
      acc += f_scalar<OP>(a.x) + f_scalar<OP>(a.y) + f_scalar<OP>(a.z) + f_scalar<OP>(a.w);
    }
  }
  // unaligned head and tail, unit by unit
  const int64_t n_tail = sp.units - sp.tail_begin;
  for (int64_t j = tid; j < sp.head + n_tail; j += stride) {
    const int64_t u = j < sp.head ? j : sp.tail_begin + (j - sp.head);
    if (OP == SO_SAMPLE_MEAN_EIKONAL)
      acc += eik_row(x[3 * u], x[3 * u + 1], x[3 * u + 2]);
    else
      acc += f_scalar<OP>(x[u]);
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0) partials[blockIdx.x] = acc;
}

__global__ void __launch_bounds__(kMaxPartials) sample_mean_final_kernel(const double* __restrict__ partials, int n_part,
                                                                         int64_t count, float* __restrict__ out) {
  __shared__ double sh[32];
  const double v = block_sum((int)threadIdx.x < n_part ? partials[threadIdx.x] : 0.0, sh);
  if (threadIdx.x == 0) out[0] = (float)(v / (double)count);
}

template <int OP>
__global__ void __launch_bounds__(kThreads) sample_mean_backward_kernel(const float* __restrict__ x, Split sp,
                                                                        const float* __restrict__ g_out, int64_t count,
                                                                        float* __restrict__ gx) {
  const float s = (float)((double)__ldg(g_out) / (double)count);
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
      __stcs(o + i, make_float4(df_scalar<OP>(a.x, s), df_scalar<OP>(a.y, s), df_scalar<OP>(a.z, s), df_scalar<OP>(a.w, s)));
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
      gx[u] = df_scalar<OP>(x[u], s);
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
void launch_forward(const float* x, int64_t n, double* ws, float* out, cudaStream_t st) {
  const Split sp = make_split<OP>(x, n, true);
  const unsigned grid = grid_for(sp);
  sample_mean_partial_kernel<OP><<<grid, kThreads, 0, st>>>(x, sp, ws);
  sample_mean_final_kernel<<<1, kMaxPartials, 0, st>>>(ws, (int)grid, sp.units, out);
}

template <int OP>
void launch_backward(const float* x, int64_t n, const float* g_out, float* gx, cudaStream_t st) {
  // 128-bit words of x and grad_x line up only when both sit at the same offset inside a word
  const bool vec = (((uintptr_t)x ^ (uintptr_t)gx) & 15) == 0;
  const Split sp = make_split<OP>(x, n, vec);
  sample_mean_backward_kernel<OP><<<grid_for(sp), kThreads, 0, st>>>(x, sp, g_out, sp.units, gx);
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
