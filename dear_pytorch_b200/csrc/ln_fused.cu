// ln_fused.cu — fused dropout + residual add + LayerNorm, forward and backward.
//
//   forward :  s = residual + dropout(a, p);  y = (s - mean(s)) * rstd(s) * gamma + beta
//   backward:  ds = LN'(dy);  d_residual = ds;  d_a = ds * mask / (1 - p);  dgamma, dbeta
//
// The transformer layer of the reference's BERT benchmark (transformers' BertSelfOutput / BertOutput,
// dear/bert_benchmark.py:60-75) runs dropout, add and LayerNorm as three ATen kernels forward and
// four to five backward, each a full pass over the [tokens, hidden] activation.  At the benchmark's
// size (2048 tokens x 1024) every one of them is a few microseconds of launch + DRAM latency, so
// the step is bound by the NUMBER of such kernels; here the forward is one kernel and the backward
// is one kernel plus a tiny column reduction.
//
// Mapping: one warp per row.  A lane owns VEC consecutive columns (one 128-bit vector) every
// 32*VEC columns, so a 1024-wide bf16 row is 4 vectors per lane, all kept in registers between the
// statistics and the normalisation: x and a are read once, s / y / mask written once.  Row statistics
// are two warp-shuffle reductions (mean, then centred second moment: no E[x^2]-E[x]^2 cancellation).
// Dropout uses Philox4x32-10 keyed by (seed, element index / 4) with the generator's graph-safe
// offset, so a captured CUDA graph draws fresh masks on every replay.
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <ATen/cuda/CUDAGraphsUtils.cuh>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <curand_kernel.h>
#include <torch/extension.h>

#include <atomic>

namespace dear {
namespace ln {

constexpr int kWarpsPerBlock = 8;
constexpr int kThreads = kWarpsPerBlock * 32;
constexpr int kMaxCols = 1024;            // widest row kept in registers (32 columns per lane)
static std::atomic<int64_t> g_launches{0};
int64_t ln_launches() { return g_launches.load(); }

template <typename T> struct Vec;
template <> struct Vec<float> {
  static constexpr int N = 4;
  static constexpr int ITERS = kMaxCols / (32 * 4);
  __device__ static float round(float f) { return f; }
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
  static constexpr int ITERS = kMaxCols / (32 * 8);
  __device__ static float round(float f) { return __bfloat162float(__float2bfloat16_rn(f)); }
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

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// keep-mask bits for the VEC elements starting at linear element index e0 (a multiple of 4)
template <int VEC>
__device__ __forceinline__ void draw_keep(uint64_t seed, uint64_t offset, uint64_t e0, float p, bool* keep) {
#pragma unroll
  for (int q = 0; q < VEC / 4; ++q) {
    curandStatePhilox4_32_10_t st;
    curand_init(seed, e0 / 4 + q, offset, &st);
    const float4 r = curand_uniform4(&st);
    keep[4 * q + 0] = r.x > p; keep[4 * q + 1] = r.y > p; keep[4 * q + 2] = r.z > p; keep[4 * q + 3] = r.w > p;
  }
}

// ------------------------------------------------------------------------------------------ forward
template <typename T, bool DROP>
__global__ void __launch_bounds__(kThreads)
ln_fwd_kernel(const T* __restrict__ a, const T* __restrict__ a_bias, const T* __restrict__ res, const T* __restrict__ gamma,
              const T* __restrict__ beta, T* __restrict__ y, T* __restrict__ s_out, float* __restrict__ mean_out,
              float* __restrict__ rstd_out, uint8_t* __restrict__ mask, int rows, int H, float eps, float p,
              at::PhiloxCudaState rng) {
  constexpr int VEC = Vec<T>::N;
  constexpr int kMaxIters = Vec<T>::ITERS;
  const int lane = threadIdx.x & 31;
  const int warp = blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  const int nwarps = gridDim.x * kWarpsPerBlock;
  uint64_t seed = 0, offset = 0;
  if (DROP) {
    auto so = at::cuda::philox::unpack(rng);
    seed = std::get<0>(so);
    offset = std::get<1>(so);
  }
  const float scale = DROP ? 1.0f / (1.0f - p) : 1.0f;
  const float inv_h = 1.0f / static_cast<float>(H);
  for (int row = warp; row < rows; row += nwarps) {
    const size_t base = static_cast<size_t>(row) * H;
    float v[kMaxIters][VEC];
    float sum = 0.f;
#pragma unroll
    for (int it = 0; it < kMaxIters; ++it) {
      const int c = (it * 32 + lane) * VEC;
      if (c < H) {
        float fa[VEC], fr[VEC];
        Vec<T>::load(a + base + c, fa);
        Vec<T>::load(res + base + c, fr);
        if (a_bias != nullptr) {                     // bias of the linear layer that produced a (its GEMM ran bias-free)
          float fb[VEC];
          Vec<T>::load(a_bias + c, fb);
#pragma unroll
          for (int i = 0; i < VEC; ++i) fa[i] = Vec<T>::round(fa[i] + fb[i]);
        }
        if (DROP) {
          bool keep[VEC];
          draw_keep<VEC>(seed, offset, base + c, p, keep);
          __align__(8) uint8_t m[VEC];
#pragma unroll
          for (int i = 0; i < VEC; ++i) {
            m[i] = keep[i] ? 1 : 0;
            fa[i] = keep[i] ? fa[i] * scale : 0.f;
          }
          if (VEC == 8) {
            *reinterpret_cast<uint2*>(mask + base + c) = *reinterpret_cast<const uint2*>(m);
          } else {
            *reinterpret_cast<uint32_t*>(mask + base + c) = *reinterpret_cast<const uint32_t*>(m);
          }
        }
        // the backward normalises the STORED s: take the statistics of the value rounded to T
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          v[it][i] = Vec<T>::round(fa[i] + fr[i]);
          sum += v[it][i];
        }
        Vec<T>::store(s_out + base + c, v[it]);
      }
    }
    const float mean = warp_sum(sum) * inv_h;
    float sq = 0.f;
#pragma unroll
    for (int it = 0; it < kMaxIters; ++it) {
      const int c = (it * 32 + lane) * VEC;
      if (c < H) {
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          const float d = v[it][i] - mean;
          sq += d * d;
        }
      }
    }
    const float rstd = rsqrtf(warp_sum(sq) * inv_h + eps);
    if (lane == 0) {
      mean_out[row] = mean;
      rstd_out[row] = rstd;
    }
#pragma unroll
    for (int it = 0; it < kMaxIters; ++it) {
      const int c = (it * 32 + lane) * VEC;
      if (c < H) {
        float g[VEC], b[VEC], o[VEC];
        Vec<T>::load(gamma + c, g);
        Vec<T>::load(beta + c, b);
#pragma unroll
        for (int i = 0; i < VEC; ++i) o[i] = (v[it][i] - mean) * rstd * g[i] + b[i];
        Vec<T>::store(y + base + c, o);
      }
    }
  }
}

// ----------------------------------------------------------------------------------------- backward
// ds, da per row; per-block partial dgamma / dbeta (/ dbias = column sums of da) to part[2 or 3][gridDim.x][H]
template <typename T, bool DROP, bool DBIAS>
__global__ void __launch_bounds__(kThreads)
ln_bwd_kernel(const T* __restrict__ dy, const T* __restrict__ s, const float* __restrict__ mean_in,
              const float* __restrict__ rstd_in, const T* __restrict__ gamma, const uint8_t* __restrict__ mask,
              T* __restrict__ ds_out, T* __restrict__ da_out, float* __restrict__ part, int rows, int H, float p) {
  constexpr int VEC = Vec<T>::N;
  constexpr int kMaxIters = Vec<T>::ITERS;
  __shared__ float red[kWarpsPerBlock][32 * VEC + 1];
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int warp = blockIdx.x * kWarpsPerBlock + wib;
  const int nwarps = gridDim.x * kWarpsPerBlock;
  const float scale = DROP ? 1.0f / (1.0f - p) : 1.0f;
  const float inv_h = 1.0f / static_cast<float>(H);
  float acc_g[kMaxIters][VEC], acc_b[kMaxIters][VEC], acc_a[DBIAS ? kMaxIters : 1][VEC];
#pragma unroll
  for (int it = 0; it < kMaxIters; ++it) {
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      acc_g[it][i] = 0.f; acc_b[it][i] = 0.f;
      if (DBIAS) acc_a[it][i] = 0.f;
    }
  }
  for (int row = warp; row < rows; row += nwarps) {
    const size_t base = static_cast<size_t>(row) * H;
    const float mean = mean_in[row], rstd = rstd_in[row];
    float xh[kMaxIters][VEC], gy[kMaxIters][VEC];
    float c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int it = 0; it < kMaxIters; ++it) {
      const int c = (it * 32 + lane) * VEC;
      if (c < H) {
        float fd[VEC], fs[VEC], g[VEC];
        Vec<T>::load(dy + base + c, fd);
        Vec<T>::load(s + base + c, fs);
        Vec<T>::load(gamma + c, g);                  // L1-resident after the first row
#pragma unroll
        for (int i = 0; i < VEC; ++i) {
          xh[it][i] = (fs[i] - mean) * rstd;
          gy[it][i] = fd[i] * g[i];
          c1 += gy[it][i];
          c2 += gy[it][i] * xh[it][i];
          acc_g[it][i] += fd[i] * xh[it][i];
          acc_b[it][i] += fd[i];
        }
      }
    }
    c1 = warp_sum(c1) * inv_h;
    c2 = warp_sum(c2) * inv_h;
#pragma unroll
    for (int it = 0; it < kMaxIters; ++it) {
      const int c = (it * 32 + lane) * VEC;
      if (c < H) {
        float o[VEC];
#pragma unroll
        for (int i = 0; i < VEC; ++i) o[i] = rstd * (gy[it][i] - c1 - xh[it][i] * c2);
        Vec<T>::store(ds_out + base + c, o);
        if (DROP) {
          __align__(8) uint8_t m[VEC];
          if (VEC == 8) {
            *reinterpret_cast<uint2*>(m) = *reinterpret_cast<const uint2*>(mask + base + c);
          } else {
            *reinterpret_cast<uint32_t*>(m) = *reinterpret_cast<const uint32_t*>(mask + base + c);
          }
#pragma unroll
          for (int i = 0; i < VEC; ++i) o[i] = m[i] ? o[i] * scale : 0.f;
          Vec<T>::store(da_out + base + c, o);
        }
        if (DBIAS) {
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc_a[it][i] += o[i];
        }
      }
    }
  }
  // block reduction of the per-warp column partials, one vector slot ("it") at a time
#pragma unroll
  for (int it = 0; it < kMaxIters; ++it) {
    if (it * 32 * VEC >= H) break;
    for (int which = 0; which < (DBIAS ? 3 : 2); ++which) {
      __syncthreads();
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        red[wib][lane * VEC + i] = which == 0 ? acc_g[it][i] : (which == 1 ? acc_b[it][i] : acc_a[DBIAS ? it : 0][i]);
      }
      __syncthreads();
      float* dst = part + (static_cast<size_t>(which) * gridDim.x + blockIdx.x) * H;
      for (int j = threadIdx.x; j < 32 * VEC; j += kThreads) {
        const int c = it * 32 * VEC + j;
        if (c < H) {
          float t = 0.f;
#pragma unroll
          for (int w = 0; w < kWarpsPerBlock; ++w) t += red[w][j];
          dst[c] = t;
        }
      }
    }
  }
}

// out[k][c] = sum_b part[k][b][c] for k < nout (dgamma, dbeta[, dbias]).  Block = 32 columns x 16 partial-row groups.
template <typename T>
__global__ void __launch_bounds__(512)
colsum_finalize(const float* __restrict__ part, T* __restrict__ out0, T* __restrict__ out1, T* __restrict__ out2,
                int nout, int nblocks, int H) {
  __shared__ float sm[3][16][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  float t[3] = {0.f, 0.f, 0.f};
  if (c < H) {
    for (int k = 0; k < nout; ++k) {
      const float* p = part + static_cast<size_t>(k) * nblocks * H + c;
#pragma unroll 4
      for (int b = threadIdx.y; b < nblocks; b += 16) t[k] += p[static_cast<size_t>(b) * H];
    }
  }
  for (int k = 0; k < nout; ++k) sm[k][threadIdx.y][threadIdx.x] = t[k];
  __syncthreads();
  if (threadIdx.y == 0 && c < H) {
    T* outs[3] = {out0, out1, out2};
    for (int k = 0; k < nout; ++k) {
      float v = t[k];
#pragma unroll
      for (int j = 1; j < 16; ++j) v += sm[k][j][threadIdx.x];
      if (sizeof(T) == 4) {
        reinterpret_cast<float*>(outs[k])[c] = v;
      } else {
        reinterpret_cast<__nv_bfloat16*>(outs[k])[c] = __float2bfloat16_rn(v);
      }
    }
  }
}

// ---------------------------------------------------------------------------- bias + GELU (elementwise)
//   forward :  h = gelu(z + b)                      (z: bias-free GEMM output, b: [N])
//   backward:  dz = dh * gelu'(z + b),  db = column sums of dz      -- one pass, instead of GeluBackward + a reduction
// Thread (tx, ty) of a 64x4 block owns one 128-bit column vector and walks rows ty, ty + 4*gridDim.y, ...
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float dgelu_erf(float x) {
  return 0.5f * (1.0f + erff(x * 0.70710678118654752440f)) + x * 0.39894228040143267794f * __expf(-0.5f * x * x);
}

template <typename T>
__global__ void __launch_bounds__(256)
bias_gelu_fwd_kernel(const T* __restrict__ z, const T* __restrict__ bias, T* __restrict__ h, int rows, int N) {
  constexpr int VEC = Vec<T>::N;
  const int c = (blockIdx.x * 64 + threadIdx.x) * VEC;
  if (c >= N) return;
  float fb[VEC];
  Vec<T>::load(bias + c, fb);
  for (int r = blockIdx.y * 4 + threadIdx.y; r < rows; r += gridDim.y * 4) {
    float f[VEC];
    Vec<T>::load(z + static_cast<size_t>(r) * N + c, f);
#pragma unroll
    for (int i = 0; i < VEC; ++i) f[i] = gelu_erf(Vec<T>::round(f[i] + fb[i]));
    Vec<T>::store(h + static_cast<size_t>(r) * N + c, f);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
bias_gelu_bwd_kernel(const T* __restrict__ dh, const T* __restrict__ z, const T* __restrict__ bias, T* __restrict__ dz,
                     float* __restrict__ part, int rows, int N) {
  constexpr int VEC = Vec<T>::N;
  __shared__ float red[4][64 * VEC + 1];
  const int c = (blockIdx.x * 64 + threadIdx.x) * VEC;
  float acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
  if (c < N) {
    float fb[VEC];
    Vec<T>::load(bias + c, fb);
    for (int r = blockIdx.y * 4 + threadIdx.y; r < rows; r += gridDim.y * 4) {
      float fz[VEC], fd[VEC];
      Vec<T>::load(z + static_cast<size_t>(r) * N + c, fz);
      Vec<T>::load(dh + static_cast<size_t>(r) * N + c, fd);
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        fd[i] = Vec<T>::round(fd[i] * dgelu_erf(Vec<T>::round(fz[i] + fb[i])));
        acc[i] += fd[i];                             // the bias gradient sums the values the weight gradient sees
      }
      Vec<T>::store(dz + static_cast<size_t>(r) * N + c, fd);
    }
  }
#pragma unroll
  for (int i = 0; i < VEC; ++i) red[threadIdx.y][threadIdx.x * VEC + i] = acc[i];
  __syncthreads();
  for (int j = threadIdx.y * 64 + threadIdx.x; j < 64 * VEC; j += 256) {
    const int cc = blockIdx.x * 64 * VEC + j;
    if (cc < N) part[static_cast<size_t>(blockIdx.y) * N + cc] = red[0][j] + red[1][j] + red[2][j] + red[3][j];
  }
}

// ------------------------------------------------------------------------------------------- host
// Every operand the kernels read or write moves as 128-bit vectors: a contiguous view at an odd storage offset is not one.
static bool aligned16(const torch::Tensor& t) { return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0; }
static bool aligned16(const c10::optional<torch::Tensor>& t) { return !t.has_value() || aligned16(*t); }

static bool ln_shape_ok(const torch::Tensor& x) {
  if (!x.is_cuda() || x.dim() < 2 || !aligned16(x)) return false;
  const int64_t H = x.size(-1);
  if (x.scalar_type() == at::kBFloat16) return H % 8 == 0 && H <= kMaxCols;
  if (x.scalar_type() == at::kFloat) return H % 4 == 0 && H <= kMaxCols;
  return false;
}

bool ln_supported(const torch::Tensor& x, const c10::optional<torch::Tensor>& residual, const c10::optional<torch::Tensor>& gamma,
                  const c10::optional<torch::Tensor>& beta, const c10::optional<torch::Tensor>& a_bias) {
  return ln_shape_ok(x) && aligned16(residual) && aligned16(gamma) && aligned16(beta) && aligned16(a_bias);
}

static int grid_for(int rows, int ctas_per_sm) {
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int want = (rows + kWarpsPerBlock - 1) / kWarpsPerBlock;
  return std::max(1, std::min(want, sms * ctas_per_sm));
}

template <typename T>
static void fwd_launch(const torch::Tensor& a, const c10::optional<torch::Tensor>& a_bias, const torch::Tensor& res, const torch::Tensor& gamma,
                       const torch::Tensor& beta, torch::Tensor& y, torch::Tensor& s, torch::Tensor& mean,
                       torch::Tensor& rstd, torch::Tensor& mask, int rows, int H, float eps, float p, bool drop) {
  auto stream = at::cuda::getCurrentCUDAStream().stream();
  const int grid = grid_for(rows, 2);
  at::PhiloxCudaState rng;
  if (drop) {
    auto gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(c10::nullopt, at::cuda::detail::getDefaultCUDAGenerator());
    std::lock_guard<std::mutex> lock(gen->mutex_);
    rng = gen->philox_cuda_state(4);        // each Philox subsequence (element index / 4) draws one float4
  }
  const T* pa = reinterpret_cast<const T*>(a.data_ptr());
  const T* pab = a_bias.has_value() ? reinterpret_cast<const T*>(a_bias->data_ptr()) : nullptr;
  const T* pr = reinterpret_cast<const T*>(res.data_ptr());
  const T* pg = reinterpret_cast<const T*>(gamma.data_ptr());
  const T* pb = reinterpret_cast<const T*>(beta.data_ptr());
  T* py = reinterpret_cast<T*>(y.data_ptr());
  T* ps = reinterpret_cast<T*>(s.data_ptr());
  if (drop) {
    ln_fwd_kernel<T, true><<<grid, kThreads, 0, stream>>>(pa, pab, pr, pg, pb, py, ps, mean.data_ptr<float>(),
                                                          rstd.data_ptr<float>(), mask.data_ptr<uint8_t>(), rows, H, eps, p, rng);
  } else {
    ln_fwd_kernel<T, false><<<grid, kThreads, 0, stream>>>(pa, pab, pr, pg, pb, py, ps, mean.data_ptr<float>(),
                                                           rstd.data_ptr<float>(), nullptr, rows, H, eps, 0.f, rng);
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  g_launches.fetch_add(1);
}

// returns {y, s, mean, rstd, mask}; mask is an empty tensor when no dropout was applied
std::vector<torch::Tensor> ln_forward(const torch::Tensor& a, const torch::Tensor& residual, const torch::Tensor& gamma,
                                      const torch::Tensor& beta, double p, bool training, double eps,
                                      const c10::optional<torch::Tensor>& a_bias) {
  TORCH_CHECK(ln_supported(a, residual, gamma, beta, a_bias),
              "dropout_add_layer_norm: unsupported tensor (16-byte aligned CUDA bf16 with H % 8 == 0 or fp32 with H % 4 == 0, H <= 1024)");
  TORCH_CHECK(a.is_contiguous() && residual.is_contiguous() && gamma.is_contiguous() && beta.is_contiguous(),
              "dropout_add_layer_norm: contiguous tensors expected");
  TORCH_CHECK(a.sizes() == residual.sizes() && a.scalar_type() == residual.scalar_type() &&
              gamma.scalar_type() == a.scalar_type() && beta.scalar_type() == a.scalar_type(), "dropout_add_layer_norm: dtype/shape mismatch");
  const int H = a.size(-1);
  TORCH_CHECK(gamma.numel() == H && beta.numel() == H, "dropout_add_layer_norm: weight/bias size");
  TORCH_CHECK(!a_bias.has_value() || (a_bias->numel() == H && a_bias->scalar_type() == a.scalar_type() && a_bias->is_contiguous()),
              "dropout_add_layer_norm: branch bias must be a contiguous [H] tensor of the activation dtype");
  TORCH_CHECK(p >= 0.0 && p < 1.0, "dropout probability must be in [0, 1)");
  c10::cuda::CUDAGuard guard(a.device());
  const int rows = a.numel() / H;
  const bool drop = training && p > 0.0;
  auto y = torch::empty_like(a);
  auto s = torch::empty_like(a);
  auto fopt = a.options().dtype(at::kFloat);
  auto mean = torch::empty({rows}, fopt);
  auto rstd = torch::empty({rows}, fopt);
  auto mask = drop ? torch::empty(a.sizes(), a.options().dtype(at::kByte)) : torch::empty({0}, a.options().dtype(at::kByte));
  if (rows > 0) {
    if (a.scalar_type() == at::kFloat) {
      fwd_launch<float>(a, a_bias, residual, gamma, beta, y, s, mean, rstd, mask, rows, H, eps, p, drop);
    } else {
      fwd_launch<__nv_bfloat16>(a, a_bias, residual, gamma, beta, y, s, mean, rstd, mask, rows, H, eps, p, drop);
    }
  }
  return {y, s, mean, rstd, mask};
}

template <typename T>
static void bwd_launch(const torch::Tensor& dy, const torch::Tensor& s, const torch::Tensor& mean, const torch::Tensor& rstd,
                       const torch::Tensor& gamma, const torch::Tensor& mask, torch::Tensor& ds, torch::Tensor& da,
                       torch::Tensor& dgamma, torch::Tensor& dbeta, torch::Tensor& dbias, int rows, int H, float p, bool drop,
                       bool want_dbias) {
  auto stream = at::cuda::getCurrentCUDAStream().stream();
  const int grid = grid_for(rows, 1);      // one partial row per CTA and reduced quantity
  const int nout = want_dbias ? 3 : 2;
  auto part = torch::empty({nout, grid, H}, dy.options().dtype(at::kFloat));
  const T* pdy = reinterpret_cast<const T*>(dy.data_ptr());
  const T* ps = reinterpret_cast<const T*>(s.data_ptr());
  const T* pg = reinterpret_cast<const T*>(gamma.data_ptr());
  T* pds = reinterpret_cast<T*>(ds.data_ptr());
  T* pda = drop ? reinterpret_cast<T*>(da.data_ptr()) : nullptr;
  const uint8_t* pm = drop ? mask.data_ptr<uint8_t>() : nullptr;
  const float* pmean = mean.data_ptr<float>();
  const float* prstd = rstd.data_ptr<float>();
  float* pp = part.data_ptr<float>();
#define DEAR_LN_BWD(DROP, DBIAS) \
  ln_bwd_kernel<T, DROP, DBIAS><<<grid, kThreads, 0, stream>>>(pdy, ps, pmean, prstd, pg, pm, pds, pda, pp, rows, H, p)
  if (drop) { if (want_dbias) DEAR_LN_BWD(true, true); else DEAR_LN_BWD(true, false); }
  else      { if (want_dbias) DEAR_LN_BWD(false, true); else DEAR_LN_BWD(false, false); }
#undef DEAR_LN_BWD
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  colsum_finalize<T><<<(H + 31) / 32, dim3(32, 16), 0, stream>>>(
      pp, reinterpret_cast<T*>(dgamma.data_ptr()), reinterpret_cast<T*>(dbeta.data_ptr()),
      want_dbias ? reinterpret_cast<T*>(dbias.data_ptr()) : nullptr, nout, grid, H);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  g_launches.fetch_add(2);
}

// returns {d_residual, d_a, dgamma, dbeta, dbias}; d_a aliases d_residual when no dropout was applied; dbias (the
// column sums of d_a, i.e. the gradient of the branch bias) is empty unless want_dbias
std::vector<torch::Tensor> ln_backward(const torch::Tensor& dy, const torch::Tensor& s, const torch::Tensor& mean,
                                       const torch::Tensor& rstd, const torch::Tensor& gamma, const torch::Tensor& mask, double p,
                                       bool want_dbias) {
  TORCH_CHECK(ln_supported(dy, s, gamma, c10::nullopt, c10::nullopt) && dy.is_contiguous() && s.is_contiguous() &&
                  s.sizes() == dy.sizes() && s.scalar_type() == dy.scalar_type(),
              "dropout_add_layer_norm backward: unsupported tensor");
  c10::cuda::CUDAGuard guard(dy.device());
  const int H = dy.size(-1);
  const int rows = dy.numel() / H;
  const bool drop = mask.numel() > 0;
  auto ds = torch::empty_like(dy);
  auto da = drop ? torch::empty_like(dy) : ds;
  auto dgamma = torch::empty_like(gamma);
  auto dbeta = torch::empty_like(gamma);
  auto dbias = want_dbias ? torch::empty_like(gamma) : torch::empty({0}, gamma.options());
  if (rows == 0) {
    dgamma.zero_(); dbeta.zero_(); dbias.zero_();
    return {ds, da, dgamma, dbeta, dbias};
  }
  if (dy.scalar_type() == at::kFloat) {
    bwd_launch<float>(dy, s, mean, rstd, gamma, mask, ds, da, dgamma, dbeta, dbias, rows, H, p, drop, want_dbias);
  } else {
    bwd_launch<__nv_bfloat16>(dy, s, mean, rstd, gamma, mask, ds, da, dgamma, dbeta, dbias, rows, H, p, drop, want_dbias);
  }
  return {ds, da, dgamma, dbeta, dbias};
}

// ---- bias + GELU ------------------------------------------------------------------------------------
static bool bg_supported(const torch::Tensor& z) {
  if (!z.is_cuda() || z.dim() < 2 || !z.is_contiguous() || !aligned16(z)) return false;
  const int64_t N = z.size(-1);
  return (z.scalar_type() == at::kBFloat16 && N % 8 == 0) || (z.scalar_type() == at::kFloat && N % 4 == 0);
}
bool bias_gelu_supported(const torch::Tensor& z, const c10::optional<torch::Tensor>& bias) {
  return bg_supported(z) && aligned16(bias);
}

static dim3 bg_grid(int rows, int N, int vec) {
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  const int gx = (N / vec + 63) / 64;
  const int gy = std::max(1, std::min((rows + 3) / 4, std::max(1, 2 * sms / gx)));
  return dim3(gx, gy);
}

torch::Tensor bias_gelu_forward(const torch::Tensor& z, const torch::Tensor& bias) {
  TORCH_CHECK(bg_supported(z), "bias_gelu: unsupported tensor (contiguous CUDA bf16 / fp32, last dim a multiple of one 128-bit vector)");
  TORCH_CHECK(bias.is_contiguous() && aligned16(bias) && bias.numel() == z.size(-1) && bias.scalar_type() == z.scalar_type(),
              "bias_gelu: bias");
  c10::cuda::CUDAGuard guard(z.device());
  const int N = z.size(-1);
  const int rows = z.numel() / N;
  auto h = torch::empty_like(z);
  if (rows == 0) return h;
  auto stream = at::cuda::getCurrentCUDAStream().stream();
  if (z.scalar_type() == at::kFloat) {
    bias_gelu_fwd_kernel<float><<<bg_grid(rows, N, 4), dim3(64, 4), 0, stream>>>(
        z.data_ptr<float>(), bias.data_ptr<float>(), h.data_ptr<float>(), rows, N);
  } else {
    using B = __nv_bfloat16;
    bias_gelu_fwd_kernel<B><<<bg_grid(rows, N, 8), dim3(64, 4), 0, stream>>>(
        reinterpret_cast<const B*>(z.data_ptr()), reinterpret_cast<const B*>(bias.data_ptr()), reinterpret_cast<B*>(h.data_ptr()), rows, N);
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  g_launches.fetch_add(1);
  return h;
}

// returns {dz, dbias}
std::vector<torch::Tensor> bias_gelu_backward(const torch::Tensor& dh, const torch::Tensor& z, const torch::Tensor& bias) {
  TORCH_CHECK(bg_supported(z) && dh.is_contiguous() && aligned16(dh) && dh.sizes() == z.sizes() && dh.scalar_type() == z.scalar_type(),
              "bias_gelu backward: unsupported tensors");
  TORCH_CHECK(bias.is_contiguous() && aligned16(bias) && bias.numel() == z.size(-1) && bias.scalar_type() == z.scalar_type(),
              "bias_gelu backward: bias");
  c10::cuda::CUDAGuard guard(z.device());
  const int N = z.size(-1);
  const int rows = z.numel() / N;
  auto dz = torch::empty_like(z);
  auto dbias = torch::empty_like(bias);
  if (rows == 0) { dbias.zero_(); return {dz, dbias}; }
  auto stream = at::cuda::getCurrentCUDAStream().stream();
  const bool f32 = z.scalar_type() == at::kFloat;
  const dim3 grid = bg_grid(rows, N, f32 ? 4 : 8);
  auto part = torch::empty({static_cast<long>(grid.y), N}, z.options().dtype(at::kFloat));
  if (f32) {
    bias_gelu_bwd_kernel<float><<<grid, dim3(64, 4), 0, stream>>>(dh.data_ptr<float>(), z.data_ptr<float>(), bias.data_ptr<float>(),
                                                                  dz.data_ptr<float>(), part.data_ptr<float>(), rows, N);
    colsum_finalize<float><<<(N + 31) / 32, dim3(32, 16), 0, stream>>>(part.data_ptr<float>(), dbias.data_ptr<float>(), nullptr,
                                                                       nullptr, 1, grid.y, N);
  } else {
    using B = __nv_bfloat16;
    bias_gelu_bwd_kernel<B><<<grid, dim3(64, 4), 0, stream>>>(
        reinterpret_cast<const B*>(dh.data_ptr()), reinterpret_cast<const B*>(z.data_ptr()), reinterpret_cast<const B*>(bias.data_ptr()),
        reinterpret_cast<B*>(dz.data_ptr()), part.data_ptr<float>(), rows, N);
    colsum_finalize<B><<<(N + 31) / 32, dim3(32, 16), 0, stream>>>(part.data_ptr<float>(), reinterpret_cast<B*>(dbias.data_ptr()),
                                                                   nullptr, nullptr, 1, grid.y, N);
  }
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  g_launches.fetch_add(2);
  return {dz, dbias};
}

}  // namespace ln
}  // namespace dear
