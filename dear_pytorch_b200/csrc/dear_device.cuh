// dear_device.cuh — device-side helpers shared by the fused kernels (kernels.cu, rs_pipe.cu):
// system-scope flag protocol, streaming loads/stores, NVLS multimem wrappers, element packing.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include "dear_common.h"

namespace dear {

constexpr int kThreads = 512;
constexpr int kMaxSmemSegs = 384;     // PackSeg entries cached in shared memory (12 KiB)
constexpr int kMaxSmemHyper = 256;    // HyperSeg entries cached in shared memory (8 KiB)

// ----------------------------------------------------------------------------
// PTX helpers
// ----------------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// 128-bit load that does not allocate in L1 (peer data is never re-read).
__device__ __forceinline__ uint4 ld_stream(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
// 128-bit load of PEER memory.  Peer addresses bypass the local L2 and are cached in L1 only (the allocating form is
// used rather than L1::no_allocate; tools/p2p_probe.cu compares the two).  Every peer address is read once per kernel
// and L1 is invalidated at kernel boundaries, so there is no staleness to worry about.
__device__ __forceinline__ uint4 ld_peer(const void* p) {
  uint4 v;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_stream(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
// NVLS: the switch reduces the same offset of every bound device and returns the sum.
__device__ __forceinline__ uint4 multimem_ld_reduce_f32(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 multimem_ld_reduce_bf16(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 multimem_ld_reduce_f16(const void* mc) {
  uint4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
// NVLS: one store, replicated by the switch into every bound device.
__device__ __forceinline__ void multimem_st(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc),
               "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

__device__ __forceinline__ uint32_t* flag_at(void* sig_base, uint32_t chan, int src) {
  return reinterpret_cast<uint32_t*>(sig_base) + size_t(chan) * kMaxRanks + src;
}

// Bounded spin until *f >= epoch (wrap-safe).  Returns false on timeout.
__device__ __forceinline__ bool wait_flag(const uint32_t* f, uint32_t epoch, uint64_t timeout_ns,
                                          uint32_t* status, uint32_t code) {
  uint32_t spins = 0;
  uint64_t t0 = 0;
  while (static_cast<int32_t>(ld_acquire_sys(f) - epoch) < 0) {
    ++spins;
    if (spins > 64) __nanosleep(64);
    if ((spins & 0xfff) == 0) {
      uint64_t now = globaltimer_ns();
      if (t0 == 0) {
        t0 = now;
      } else if (now - t0 > timeout_ns) {
        if (status != nullptr) {
          *reinterpret_cast<volatile uint32_t*>(status) = code;
          __threadfence_system();
        }
        return false;
      }
    }
  }
  return true;
}

// Threads [0, world) each wait for one source rank's flag, then the CTA syncs.
__device__ __forceinline__ void wait_all_peers(void* sig_local, uint32_t chan, uint32_t epoch,
                                               int world, uint64_t timeout_ns, uint32_t* status,
                                               uint32_t code) {
  if (static_cast<int>(threadIdx.x) < world)
    wait_flag(flag_at(sig_local, chan, threadIdx.x), epoch, timeout_ns, status, code);
  __syncthreads();
}

// Threads [0, world) each publish `epoch` into one peer's pad (slot = my rank).
// Must be called by the whole CTA after the data writes; includes the bar.sync.
__device__ __forceinline__ void signal_all_peers(const PeerTable& sig, uint32_t chan, int rank,
                                                 int world, uint32_t epoch) {
  if (static_cast<int>(threadIdx.x) < world) {
    __threadfence_system();
    st_release_sys(flag_at(sig.ptr[threadIdx.x], chan, rank), epoch);
  }
}

// Grid-wide arrival counter.  Returns true (CTA-uniform) for the last CTA to arrive.
__device__ __forceinline__ bool grid_arrive_is_last(uint32_t* counter) {
  __shared__ uint32_t s_is_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence_system();                        // release this CTA's writes
    uint32_t old = atomicAdd(counter, 1u);
    __threadfence();                               // acquire the other CTAs' writes
    s_is_last = (old == gridDim.x - 1) ? 1u : 0u;
  }
  __syncthreads();
  return s_is_last != 0;
}

// true when none of f[0..N) is inf or NaN (dynamic loss scaling's overflow test)
template <int N>
__device__ __forceinline__ bool all_finite(const float* f) {
  bool ok = true;
#pragma unroll
  for (int i = 0; i < N; ++i) ok &= isfinite(f[i]);
  return ok;
}

// sum of squares of f[0..N) (global-norm clipping)
template <int N>
__device__ __forceinline__ float sum_sq(const float* f) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < N; ++i) s += f[i] * f[i];
  return s;
}

// Clipping epilogue of Kernel A, called by the whole CTA before the grid-wide exit arrive: reduce the threads' sums of
// squares in a fixed order (butterfly within each warp, then the warps in index order) and store the CTA's partial.
// The same data-to-thread assignment therefore gives the same bits on every run.
__device__ __forceinline__ void clip_store_cta_partial(ClipState* clip, uint32_t slot, float ss) {
  __shared__ float s_warp[32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (uint32_t w = 0; w < (blockDim.x >> 5); ++w) t += s_warp[w];
    clip_cta_partials(clip, slot)[blockIdx.x] = t;
  }
}

// Run by thread 0 of the last CTA to arrive: the bucket's slot = its CTAs' partials summed in CTA order.
__device__ __forceinline__ void clip_combine_slot(ClipState* clip, uint32_t slot) {
  const volatile float* part = clip_cta_partials(clip, slot);
  float t = 0.f;
  for (uint32_t b = 0; b < gridDim.x; ++b) t += part[b];
  clip_slots(clip)[slot] = t;
}

// ----------------------------------------------------------------------------
// element helpers
// ----------------------------------------------------------------------------
template <typename T> struct ElemTraits;
template <> struct ElemTraits<float> {
  static constexpr int kPerVec = 4;
  __device__ static void unpack(const uint4& v, float* f) {
    f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
    f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
  }
  __device__ static uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                      __float_as_uint(f[3]));
  }
  __device__ static uint4 mc_reduce(const void* mc) { return multimem_ld_reduce_f32(mc); }
  __device__ static float from_raw16(uint16_t) { return 0.f; }   // (not a 16-bit type)
  __device__ static uint16_t to_raw16(float) { return 0; }
};
template <> struct ElemTraits<__nv_bfloat16> {
  static constexpr int kPerVec = 8;
  __device__ static void unpack(const uint4& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  __device__ static uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
  __device__ static uint4 mc_reduce(const void* mc) { return multimem_ld_reduce_bf16(mc); }
  __device__ static float from_raw16(uint16_t r) { return __uint_as_float(uint32_t(r) << 16); }
  __device__ static uint16_t to_raw16(float x) { return __bfloat16_as_ushort(__float2bfloat16_rn(x)); }
};
template <> struct ElemTraits<__half> {
  static constexpr int kPerVec = 8;
  __device__ static void unpack(const uint4& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 h = *reinterpret_cast<const __half2*>(&w[i]);
      float2 t = __half22float2(h);
      f[2 * i] = t.x; f[2 * i + 1] = t.y;
    }
  }
  __device__ static uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
  __device__ static uint4 mc_reduce(const void* mc) { return multimem_ld_reduce_f16(mc); }
  __device__ static float from_raw16(uint16_t r) { return __half2float(__ushort_as_half(r)); }
  __device__ static uint16_t to_raw16(float x) { return __half_as_ushort(__float2half_rn(x)); }
};

}  // namespace dear
