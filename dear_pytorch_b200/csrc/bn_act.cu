// bn_act.cu — fused BatchNorm2d (+ residual add) (+ ReLU), channels-last, training and inference.
//
// Why: in the ResNet-50 step, cuDNN BatchNorm forward/backward plus the separate ReLU / add elementwise kernels
// are a large share of GPU kernel time — all of it HBM-bound.  Unfused, a BN+ReLU layer costs ~13 tensor passes per
// iteration (BN fwd 3, ReLU fwd 2, ReLU bwd 3, BN bwd 5); fused it costs 8:
//     forward : stats (read x) -> finalize -> apply (read x [,z], write y)
//     backward: reduce (read dy, x [,y]) -> finalize -> apply (read dy, x [,y], write dx [,dz])
// The ReLU mask is never stored: it is recomputed from x with exactly the forward arithmetic
// (or read from y when a residual was added).
//
// Layout: x is NHWC == a row-major [M, C] matrix (M = N*H*W).  A thread owns VEC consecutive
// channels (one 128-bit vector) and walks down the rows, so per-channel parameters live in
// registers and every access is a coalesced 128-bit load/store.  Statistics use Welford's update
// per element and Chan's merge across threads / CTAs (no E[x^2]-E[x]^2 cancellation).
//
// The reference has no such op (its models are stock torchvision: BatchNorm2d + ReLU as separate
// cuDNN / ATen kernels, dear/imagenet_benchmark.py:78-82).
#include <atomic>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAStream.h>
#include <c10/cuda/CUDAGuard.h>

namespace dear {
namespace bn {

constexpr int kThreads = 256;
static std::atomic<int64_t> g_launches{0};      // kernels launched by this file (bench.py reports them)
int64_t bn_act_launches() { return g_launches.load(); }

template <typename T> struct Vec;
template <> struct Vec<float> {
  static constexpr int N = 4;
  __device__ static void load(const float* p, float* f) {
    const float4 v = *reinterpret_cast<const float4*>(p);
    f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
  }
  __device__ static void store(float* p, const float* f) {
    *reinterpret_cast<float4*>(p) = make_float4(f[0], f[1], f[2], f[3]);
  }
};
template <> struct Vec<__nv_bfloat16> {
  static constexpr int N = 8;
  __device__ static void load(const __nv_bfloat16* p, float* f) {
    const uint4 v = *reinterpret_cast<const uint4*>(p);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ static void store(__nv_bfloat16* p, const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    *reinterpret_cast<uint4*>(p) = make_uint4(w[0], w[1], w[2], w[3]);
  }
};

// Geometry shared by every kernel: TXV vectors across channels per CTA, TY rows per sweep.
struct Geo {
  int64_t M;      // rows
  int C;          // channels
  int txv;        // channel vectors per CTA (power of two, <= 64)
  int ty;         // rows per sweep = kThreads / txv
  int row_blocks; // gridDim.x
  int ch_groups;  // gridDim.y
};

// y_pre(x) — THE one definition of the pre-activation, used by forward and by the backward's mask.
__device__ __forceinline__ float pre_act(float x, float scale, float shift) { return fmaf(x, scale, shift); }

// ---------------------------------------------------------------------------------------------
// forward 1: per-CTA Welford statistics -> partial[(row_block, c)] = (mean, M2), count per block
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads) bn_stats_kernel(const T* __restrict__ x, float* __restrict__ part_mean,
                                                            float* __restrict__ part_m2, float* __restrict__ part_n,
                                                            Geo g) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];                 // [ty][txv*V] x {mean, m2} + [ty] counts
  const int tx = threadIdx.x % g.txv, ty = threadIdx.x / g.txv;
  const int c0 = (blockIdx.y * g.txv + tx) * V;
  const int64_t rows_per_block = (g.M + g.row_blocks - 1) / g.row_blocks;
  const int64_t r0 = blockIdx.x * rows_per_block;
  const int64_t r1 = min(g.M, r0 + rows_per_block);
  float mean[V], m2[V];
#pragma unroll
  for (int k = 0; k < V; ++k) { mean[k] = 0.f; m2[k] = 0.f; }
  float n = 0.f;
  for (int64_t r = r0 + ty; r < r1; r += 2 * g.ty) {
    float v[2][V];
    const bool two = r + g.ty < r1;
    Vec<T>::load(x + r * g.C + c0, v[0]);                       // both loads in flight before the
    if (two) Vec<T>::load(x + (r + g.ty) * g.C + c0, v[1]);     // dependent Welford updates
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      if (u == 1 && !two) break;
      n += 1.f;
      const float inv = 1.f / n;
#pragma unroll
      for (int k = 0; k < V; ++k) {
        const float d = v[u][k] - mean[k];
        mean[k] += d * inv;
        m2[k] = fmaf(d, v[u][k] - mean[k], m2[k]);
      }
    }
  }
  // merge the ty threads that share this channel vector (Chan et al.)
  const int width = g.txv * V;
  float* s_mean = smem;
  float* s_m2 = smem + g.ty * width;
  float* s_n = smem + 2 * g.ty * width;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    s_mean[ty * width + tx * V + k] = mean[k];
    s_m2[ty * width + tx * V + k] = m2[k];
  }
  if (tx == 0) s_n[ty] = n;
  __syncthreads();
  if (ty == 0) {
    float na = s_n[0];
    for (int j = 1; j < g.ty; ++j) {
      const float nb = s_n[j];
      if (nb > 0.f) {
        const float nab = na + nb;
#pragma unroll
        for (int k = 0; k < V; ++k) {
          const float mb = s_mean[j * width + tx * V + k];
          const float d = mb - mean[k];
          mean[k] += d * (nb / nab);
          m2[k] += s_m2[j * width + tx * V + k] + d * d * (na * nb / nab);
        }
        na = nab;
      }
    }
#pragma unroll
    for (int k = 0; k < V; ++k) {
      part_mean[int64_t(c0 + k) * g.row_blocks + blockIdx.x] = mean[k];
      part_m2[int64_t(c0 + k) * g.row_blocks + blockIdx.x] = m2[k];
    }
    if (tx == 0 && blockIdx.y == 0) part_n[blockIdx.x] = na;
  }
}

// forward 2: merge the row-block partials; one thread per channel.  Writes the saved mean / invstd,
// the folded scale / shift for the apply kernel and updates the running statistics.
__global__ void bn_finalize_kernel(const float* __restrict__ part_mean, const float* __restrict__ part_m2,
                                   const float* __restrict__ part_n, int row_blocks, int C, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, float eps, float momentum, float* running_mean,
                                   float* running_var, float* __restrict__ save_mean, float* __restrict__ save_invstd,
                                   float* __restrict__ scale, float* __restrict__ shift) {
  // ONE WARP PER CHANNEL: the lanes stride over the row-block partials (4 independent loads in
  // flight per lane — a serial loop over the partials costs one L2 round trip per iteration and was
  // measured at 26-48 us per layer), then a 5-step shuffle merge (Chan).
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;                                   // whole warps exit together
  float n = 0.f, mean = 0.f, m2 = 0.f;
  for (int b0 = lane; b0 < row_blocks; b0 += 128) {
    float nb[4], mb[4], qb[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int b = b0 + 32 * u;
      const bool ok = b < row_blocks;
      nb[u] = ok ? part_n[b] : 0.f;
      mb[u] = ok ? part_mean[int64_t(c) * row_blocks + b] : 0.f;
      qb[u] = ok ? part_m2[int64_t(c) * row_blocks + b] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (nb[u] > 0.f) {
        const float nab = n + nb[u];
        const float d = mb[u] - mean;
        mean += d * (nb[u] / nab);
        m2 += qb[u] + d * d * (n * nb[u] / nab);
        n = nab;
      }
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float nb = __shfl_down_sync(0xffffffffu, n, off);
    const float mb = __shfl_down_sync(0xffffffffu, mean, off);
    const float qb = __shfl_down_sync(0xffffffffu, m2, off);
    if (nb > 0.f) {
      const float nab = n + nb;
      const float d = mb - mean;
      mean += d * (nb / nab);
      m2 += qb + d * d * (n * nb / nab);
      n = nab;
    }
  }
  if (lane != 0) return;
  const float var = m2 / n;
  const float invstd = rsqrtf(var + eps);
  save_mean[c] = mean;
  save_invstd[c] = invstd;
  const float s = (gamma ? gamma[c] : 1.f) * invstd;
  scale[c] = s;
  shift[c] = (beta ? beta[c] : 0.f) - mean * s;
  if (running_mean != nullptr) {
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * (n > 1.f ? m2 / (n - 1.f) : var);
  }
}

// inference: fold running statistics into scale / shift.
__global__ void bn_fold_kernel(const float* __restrict__ mean, const float* __restrict__ var, const float* __restrict__ gamma,
                               const float* __restrict__ beta, float eps, int C, float* __restrict__ scale,
                               float* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const float s = (gamma ? gamma[c] : 1.f) * rsqrtf(var[c] + eps);
  scale[c] = s;
  shift[c] = (beta ? beta[c] : 0.f) - mean[c] * s;
}

// forward 3: y = act(x*scale + shift (+ z))
template <typename T, bool RELU, bool RES>
__global__ void __launch_bounds__(kThreads) bn_apply_kernel(const T* __restrict__ x, const T* __restrict__ z,
                                                            const float* __restrict__ scale, const float* __restrict__ shift,
                                                            T* __restrict__ y, Geo g) {
  constexpr int V = Vec<T>::N;
  const int tx = threadIdx.x % g.txv, ty = threadIdx.x / g.txv;
  const int c0 = (blockIdx.y * g.txv + tx) * V;
  float sc[V], sh[V];
#pragma unroll
  for (int k = 0; k < V; ++k) { sc[k] = scale[c0 + k]; sh[k] = shift[c0 + k]; }
  const int64_t stride = int64_t(g.row_blocks) * g.ty;
  for (int64_t r = int64_t(blockIdx.x) * g.ty + ty; r < g.M; r += stride) {
    float v[V], o[V];
    Vec<T>::load(x + r * g.C + c0, v);
    if (RES) {
      float zz[V];
      Vec<T>::load(z + r * g.C + c0, zz);
#pragma unroll
      for (int k = 0; k < V; ++k) o[k] = pre_act(v[k], sc[k], sh[k]) + zz[k];
    } else {
#pragma unroll
      for (int k = 0; k < V; ++k) o[k] = pre_act(v[k], sc[k], sh[k]);
    }
    if (RELU) {
#pragma unroll
      for (int k = 0; k < V; ++k) o[k] = fmaxf(o[k], 0.f);
    }
    Vec<T>::store(y + r * g.C + c0, o);
  }
}

// ---------------------------------------------------------------------------------------------
// backward 1: per-CTA partial sums  s1 = sum(g), s2 = sum(g * xhat),  g = dy * relu_mask
// ---------------------------------------------------------------------------------------------
template <typename T, bool RELU, bool RES>
__global__ void __launch_bounds__(kThreads) bn_bwd_reduce_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                 const T* __restrict__ y, const float* __restrict__ mean,
                                                                 const float* __restrict__ invstd, const float* __restrict__ scale,
                                                                 const float* __restrict__ shift, float* __restrict__ part_s1,
                                                                 float* __restrict__ part_s2, Geo g) {
  constexpr int V = Vec<T>::N;
  extern __shared__ float smem[];
  const int tx = threadIdx.x % g.txv, ty = threadIdx.x / g.txv;
  const int c0 = (blockIdx.y * g.txv + tx) * V;
  float mu[V], is[V], sc[V], sh[V], s1[V], s2[V];
#pragma unroll
  for (int k = 0; k < V; ++k) {
    mu[k] = mean[c0 + k]; is[k] = invstd[c0 + k]; sc[k] = scale[c0 + k]; sh[k] = shift[c0 + k];
    s1[k] = 0.f; s2[k] = 0.f;
  }
  const int64_t stride = int64_t(g.row_blocks) * g.ty;
  for (int64_t r = int64_t(blockIdx.x) * g.ty + ty; r < g.M; r += stride) {
    float d[V], xv[V];
    Vec<T>::load(dy + r * g.C + c0, d);
    Vec<T>::load(x + r * g.C + c0, xv);
    if (RELU) {
      if (RES) {
        float yv[V];
        Vec<T>::load(y + r * g.C + c0, yv);
#pragma unroll
        for (int k = 0; k < V; ++k) d[k] = yv[k] > 0.f ? d[k] : 0.f;
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k) d[k] = pre_act(xv[k], sc[k], sh[k]) > 0.f ? d[k] : 0.f;
      }
    }
#pragma unroll
    for (int k = 0; k < V; ++k) {
      s1[k] += d[k];
      s2[k] = fmaf(d[k], (xv[k] - mu[k]) * is[k], s2[k]);
    }
  }
  const int width = g.txv * V;
  float* a = smem;
  float* b = smem + g.ty * width;
#pragma unroll
  for (int k = 0; k < V; ++k) {
    a[ty * width + tx * V + k] = s1[k];
    b[ty * width + tx * V + k] = s2[k];
  }
  __syncthreads();
  if (ty == 0) {
    for (int j = 1; j < g.ty; ++j) {
#pragma unroll
      for (int k = 0; k < V; ++k) {
        s1[k] += a[j * width + tx * V + k];
        s2[k] += b[j * width + tx * V + k];
      }
    }
#pragma unroll
    for (int k = 0; k < V; ++k) {
      part_s1[int64_t(c0 + k) * g.row_blocks + blockIdx.x] = s1[k];
      part_s2[int64_t(c0 + k) * g.row_blocks + blockIdx.x] = s2[k];
    }
  }
}

__global__ void bn_bwd_finalize_kernel(const float* __restrict__ part_s1, const float* __restrict__ part_s2, int row_blocks,
                                       int C, float inv_m, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                       float* __restrict__ c1, float* __restrict__ c2) {
  // one warp per channel, lanes over the row-block partials, shuffle reduction (fixed order => deterministic)
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  float s1 = 0.f, s2 = 0.f;
  for (int b0 = lane; b0 < row_blocks; b0 += 128) {
    float a[4], q[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int b = b0 + 32 * u;
      const bool ok = b < row_blocks;
      a[u] = ok ? part_s1[int64_t(c) * row_blocks + b] : 0.f;
      q[u] = ok ? part_s2[int64_t(c) * row_blocks + b] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < 4; ++u) { s1 += a[u]; s2 += q[u]; }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s1 += __shfl_down_sync(0xffffffffu, s1, off);
    s2 += __shfl_down_sync(0xffffffffu, s2, off);
  }
  if (lane != 0) return;
  dgamma[c] = s2;
  dbeta[c] = s1;
  c1[c] = s1 * inv_m;
  c2[c] = s2 * inv_m;
}

// backward 3: dx = gamma*invstd * (g - c1 - xhat*c2);  dz = g
template <typename T, bool RELU, bool RES>
__global__ void __launch_bounds__(kThreads) bn_bwd_apply_kernel(const T* __restrict__ dy, const T* __restrict__ x,
                                                                const T* __restrict__ y, const float* __restrict__ mean,
                                                                const float* __restrict__ invstd, const float* __restrict__ scale,
                                                                const float* __restrict__ shift, const float* __restrict__ c1,
                                                                const float* __restrict__ c2, T* __restrict__ dx,
                                                                T* __restrict__ dz, Geo g) {
  constexpr int V = Vec<T>::N;
  const int tx = threadIdx.x % g.txv, ty = threadIdx.x / g.txv;
  const int c0 = (blockIdx.y * g.txv + tx) * V;
  float mu[V], is[V], sc[V], sh[V], k1[V], k2[V];
#pragma unroll
  for (int k = 0; k < V; ++k) {
    mu[k] = mean[c0 + k]; is[k] = invstd[c0 + k]; sc[k] = scale[c0 + k]; sh[k] = shift[c0 + k];
    k1[k] = c1[c0 + k]; k2[k] = c2[c0 + k];
  }
  const int64_t stride = int64_t(g.row_blocks) * g.ty;
  for (int64_t r = int64_t(blockIdx.x) * g.ty + ty; r < g.M; r += stride) {
    float d[V], xv[V], o[V];
    Vec<T>::load(dy + r * g.C + c0, d);
    Vec<T>::load(x + r * g.C + c0, xv);
    if (RELU) {
      if (RES) {
        float yv[V];
        Vec<T>::load(y + r * g.C + c0, yv);
#pragma unroll
        for (int k = 0; k < V; ++k) d[k] = yv[k] > 0.f ? d[k] : 0.f;
      } else {
#pragma unroll
        for (int k = 0; k < V; ++k) d[k] = pre_act(xv[k], sc[k], sh[k]) > 0.f ? d[k] : 0.f;
      }
    }
    if (RES) Vec<T>::store(dz + r * g.C + c0, d);
#pragma unroll
    for (int k = 0; k < V; ++k) o[k] = sc[k] * (d[k] - k1[k] - (xv[k] - mu[k]) * is[k] * k2[k]);
    Vec<T>::store(dx + r * g.C + c0, o);
  }
}

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static bool make_geo(int64_t M, int64_t C, int vec, Geo* g) {
  if (C % vec != 0) return false;
  const int64_t cv = C / vec;
  // channel vectors per CTA: the largest power-of-two divisor of cv (<= 64).  ResNet widths give 16..64;
  // DenseNet (C = 64 + 32k) gives 8; widths without a divisor >= 4 fall back to the PyTorch composite.
  int txv = 1;
  while (txv < 64 && cv % (int64_t(txv) * 2) == 0) txv *= 2;
  if (txv < 4) return false;
  g->M = M;
  g->C = static_cast<int>(C);
  g->txv = txv;
  g->ty = kThreads / txv;
  g->ch_groups = static_cast<int>(cv / txv);
  int64_t want = (M + int64_t(g->ty) * 8 - 1) / (int64_t(g->ty) * 8);    // >= 8 rows per thread
  const int64_t sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  int64_t cap = std::max<int64_t>(1, (sms * 8) / g->ch_groups);      // 8 x 256 threads per SM
  g->row_blocks = static_cast<int>(std::max<int64_t>(1, std::min(want, cap)));
  return true;
}

// Every activation-sized operand moves as 128-bit vectors: a contiguous view at an odd storage offset is not one.
static bool aligned16(const torch::Tensor& t) { return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0; }

static bool supported(const torch::Tensor& x) {
  if (!x.is_cuda() || x.dim() != 4) return false;
  if (x.scalar_type() != torch::kFloat && x.scalar_type() != torch::kBFloat16) return false;
  if (!x.is_contiguous(at::MemoryFormat::ChannelsLast) || !aligned16(x)) return false;
  Geo g;
  return make_geo(x.size(0) * x.size(2) * x.size(3), x.size(1), x.scalar_type() == torch::kFloat ? 4 : 8, &g);
}

bool bn_act_supported(const torch::Tensor& x, const c10::optional<torch::Tensor>& residual) {
  return supported(x) && (!residual.has_value() || aligned16(*residual));
}

template <typename T>
static void fwd_impl(const torch::Tensor& x, const c10::optional<torch::Tensor>& z, const float* scale, const float* shift,
                     torch::Tensor& y, bool relu, const Geo& g, cudaStream_t s) {
  const dim3 grid(g.row_blocks, g.ch_groups);
  const T* xp = reinterpret_cast<const T*>(x.data_ptr());
  const T* zp = z.has_value() ? reinterpret_cast<const T*>(z->data_ptr()) : nullptr;
  T* yp = reinterpret_cast<T*>(y.data_ptr());
  if (zp) {
    if (relu) bn_apply_kernel<T, true, true><<<grid, kThreads, 0, s>>>(xp, zp, scale, shift, yp, g);
    else bn_apply_kernel<T, false, true><<<grid, kThreads, 0, s>>>(xp, zp, scale, shift, yp, g);
  } else {
    if (relu) bn_apply_kernel<T, true, false><<<grid, kThreads, 0, s>>>(xp, zp, scale, shift, yp, g);
    else bn_apply_kernel<T, false, false><<<grid, kThreads, 0, s>>>(xp, zp, scale, shift, yp, g);
  }
}

// returns (y, save_mean, save_invstd, scale, shift)
std::vector<torch::Tensor> bn_act_forward(const torch::Tensor& x, const c10::optional<torch::Tensor>& z,
                                          const c10::optional<torch::Tensor>& gamma, const c10::optional<torch::Tensor>& beta,
                                          c10::optional<torch::Tensor> running_mean, c10::optional<torch::Tensor> running_var,
                                          bool training, double momentum, double eps, bool relu) {
  TORCH_CHECK(supported(x), "bn_act_forward: unsupported input (need CUDA, 4-D channels_last, fp32/bf16, power-of-two width)");
  if (z.has_value()) TORCH_CHECK(z->sizes() == x.sizes() && z->scalar_type() == x.scalar_type() &&
                                 z->is_contiguous(at::MemoryFormat::ChannelsLast) && aligned16(*z),
                                 "residual must match x (and be 16-byte aligned)");
  const int64_t M = x.size(0) * x.size(2) * x.size(3);
  // the variance of one value is undefined (and its unbiased form divides by zero); ops/fused_bn.py raises F.batch_norm's
  // ValueError before it gets here
  TORCH_CHECK(!training || M > 1, "bn_act_forward: Expected more than 1 value per channel when training");
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream().stream();
  const bool f32 = x.scalar_type() == torch::kFloat;
  Geo g;
  make_geo(M, x.size(1), f32 ? 4 : 8, &g);
  const int C = g.C;
  auto fopt = x.options().dtype(torch::kFloat).memory_format(at::MemoryFormat::Contiguous);
  auto y = torch::empty_like(x);
  auto stats = torch::empty({4, C}, fopt);          // one allocation: mean | invstd | scale | shift
  auto save_mean = stats.select(0, 0), save_invstd = stats.select(0, 1);
  auto scale = stats.select(0, 2), shift = stats.select(0, 3);
  const float* gp = gamma.has_value() ? gamma->data_ptr<float>() : nullptr;
  const float* bp = beta.has_value() ? beta->data_ptr<float>() : nullptr;
  if (training) {
    auto part = torch::empty({2 * int64_t(g.row_blocks) * C + g.row_blocks}, fopt);
    auto part_n = part.narrow(0, 2 * int64_t(g.row_blocks) * C, g.row_blocks);
    const dim3 grid(g.row_blocks, g.ch_groups);
    const int vec = f32 ? 4 : 8;
    const size_t smem = (2 * size_t(g.ty) * g.txv * vec + g.ty) * sizeof(float);
    float* pm = part.data_ptr<float>();
    float* pm2 = pm + int64_t(g.row_blocks) * C;
    if (f32) bn_stats_kernel<float><<<grid, kThreads, smem, s>>>(x.data_ptr<float>(), pm, pm2, part_n.data_ptr<float>(), g);
    else bn_stats_kernel<__nv_bfloat16><<<grid, kThreads, smem, s>>>(reinterpret_cast<const __nv_bfloat16*>(x.data_ptr()), pm, pm2,
                                                                    part_n.data_ptr<float>(), g);
    bn_finalize_kernel<<<(C + 7) / 8, 256, 0, s>>>(          // 8 warps per CTA, one warp per channel
        pm, pm2, part_n.data_ptr<float>(), g.row_blocks, C, gp, bp, static_cast<float>(eps), static_cast<float>(momentum),
        running_mean.has_value() ? running_mean->data_ptr<float>() : nullptr,
        running_var.has_value() ? running_var->data_ptr<float>() : nullptr, save_mean.data_ptr<float>(),
        save_invstd.data_ptr<float>(), scale.data_ptr<float>(), shift.data_ptr<float>());
  } else {
    TORCH_CHECK(running_mean.has_value() && running_var.has_value(), "inference needs running statistics");
    bn_fold_kernel<<<(C + 127) / 128, 128, 0, s>>>(running_mean->data_ptr<float>(), running_var->data_ptr<float>(), gp, bp,
                                                   static_cast<float>(eps), C, scale.data_ptr<float>(), shift.data_ptr<float>());
  }
  if (f32) fwd_impl<float>(x, z, scale.data_ptr<float>(), shift.data_ptr<float>(), y, relu, g, s);
  else fwd_impl<__nv_bfloat16>(x, z, scale.data_ptr<float>(), shift.data_ptr<float>(), y, relu, g, s);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  g_launches.fetch_add(training ? 3 : 2);
  return {y, save_mean, save_invstd, scale, shift};
}

template <typename T>
static void bwd_impl(const torch::Tensor& dy, const torch::Tensor& x, const c10::optional<torch::Tensor>& y,
                     const float* mean, const float* invstd, const float* scale, const float* shift, float* ps1, float* ps2,
                     float* dgamma, float* dbeta, float* c1, float* c2, torch::Tensor& dx, c10::optional<torch::Tensor>& dz,
                     bool relu, const Geo& g, cudaStream_t s) {
  const dim3 grid(g.row_blocks, g.ch_groups);
  const T* dyp = reinterpret_cast<const T*>(dy.data_ptr());
  const T* xp = reinterpret_cast<const T*>(x.data_ptr());
  const bool res = dz.has_value();
  const T* yp = (res && relu) ? reinterpret_cast<const T*>(y->data_ptr()) : nullptr;
  T* dxp = reinterpret_cast<T*>(dx.data_ptr());
  T* dzp = res ? reinterpret_cast<T*>(dz->data_ptr()) : nullptr;
  const size_t smem = 2 * size_t(g.ty) * g.txv * Vec<T>::N * sizeof(float);
#define DEAR_BN_BWD(RELU, RES)                                                                                         \
  bn_bwd_reduce_kernel<T, RELU, RES><<<grid, kThreads, smem, s>>>(dyp, xp, yp, mean, invstd, scale, shift, ps1, ps2, g); \
  bn_bwd_finalize_kernel<<<(g.C + 7) / 8, 256, 0, s>>>(ps1, ps2, g.row_blocks, g.C, 1.f / float(g.M), dgamma, dbeta, c1, c2); \
  bn_bwd_apply_kernel<T, RELU, RES><<<grid, kThreads, 0, s>>>(dyp, xp, yp, mean, invstd, scale, shift, c1, c2, dxp, dzp, g);
  if (relu && res) { DEAR_BN_BWD(true, true) }
  else if (relu) { DEAR_BN_BWD(true, false) }
  else if (res) { DEAR_BN_BWD(false, true) }
  else { DEAR_BN_BWD(false, false) }
#undef DEAR_BN_BWD
}

// returns (dx, dz or undefined, dgamma, dbeta)
std::vector<torch::Tensor> bn_act_backward(const torch::Tensor& dy_in, const torch::Tensor& x, const c10::optional<torch::Tensor>& y,
                                           const torch::Tensor& save_mean, const torch::Tensor& save_invstd,
                                           const torch::Tensor& scale, const torch::Tensor& shift, bool relu, bool has_residual) {
  TORCH_CHECK(supported(x), "bn_act_backward: unsupported input");
  auto dy = dy_in.is_contiguous(at::MemoryFormat::ChannelsLast) && aligned16(dy_in)
                ? dy_in : dy_in.clone(at::MemoryFormat::ChannelsLast);
  TORCH_CHECK(dy.scalar_type() == x.scalar_type() && dy.sizes() == x.sizes() && aligned16(dy),
              "grad dtype and shape must match the input");
  if (has_residual && relu)
    TORCH_CHECK(y.has_value() && y->sizes() == x.sizes() && y->scalar_type() == x.scalar_type() &&
                    y->is_contiguous(at::MemoryFormat::ChannelsLast) && aligned16(*y),
                "residual + ReLU backward needs the forward output");
  c10::cuda::CUDAGuard guard(x.device());
  cudaStream_t s = c10::cuda::getCurrentCUDAStream().stream();
  const bool f32 = x.scalar_type() == torch::kFloat;
  Geo g;
  make_geo(x.size(0) * x.size(2) * x.size(3), x.size(1), f32 ? 4 : 8, &g);
  const int C = g.C;
  auto fopt = x.options().dtype(torch::kFloat).memory_format(at::MemoryFormat::Contiguous);
  auto part = torch::empty({2, g.row_blocks, C}, fopt);
  auto small = torch::empty({4, C}, fopt);         // one allocation: dgamma | dbeta | c1 | c2
  auto dgamma = small.select(0, 0), dbeta = small.select(0, 1);
  auto coef = small.narrow(0, 2, 2);
  auto dx = torch::empty_like(x);
  c10::optional<torch::Tensor> dz;
  if (has_residual) dz = torch::empty_like(x);
  float* ps1 = part.data_ptr<float>();
  float* ps2 = ps1 + int64_t(g.row_blocks) * C;
  float* c1 = coef.data_ptr<float>();
  float* c2 = c1 + C;
  if (f32)
    bwd_impl<float>(dy, x, y, save_mean.data_ptr<float>(), save_invstd.data_ptr<float>(), scale.data_ptr<float>(),
                    shift.data_ptr<float>(), ps1, ps2, dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), c1, c2, dx, dz, relu, g, s);
  else
    bwd_impl<__nv_bfloat16>(dy, x, y, save_mean.data_ptr<float>(), save_invstd.data_ptr<float>(), scale.data_ptr<float>(),
                            shift.data_ptr<float>(), ps1, ps2, dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), c1, c2, dx, dz,
                            relu, g, s);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  g_launches.fetch_add(3);
  return {dx, dz.has_value() ? *dz : torch::Tensor(), dgamma, dbeta};
}

}  // namespace bn
}  // namespace dear
