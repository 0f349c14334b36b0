// p2p_probe.cu — what can one H100 pull from / push to its NVSwitch peers, and with which instruction?
//
// Single process, N devices with peer access enabled.  Every device d runs the SAME access pattern the
// fused reduce-scatter / all-gather kernels use (csrc/kernels.cu):
//   pull : out_d[i] = sum_q  bucket_q[d*shard + i]      (read (N-1)/N of a shard-set over NVLink, fp32 add)
//   push : bucket_q[d*shard + i] = shard_d[i]  for all q (write to every peer)
// and is timed with CUDA events on its own stream (max over devices is reported).  Variants:
//   pull  ldg_na : ld.global.L1::no_allocate.v4        (LDG.E.NA.128)
//         ldg    : ld.global.v4
//         tma    : cp.async.bulk global->shared (UBLKCP) ring with mbarriers, reduce from shared memory
//   push  stg_na : st.global.L1::no_allocate.v4
//         tma    : cp.async.bulk shared->global (UBLKCP) to every peer
// Build:  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -o build/p2p_probe tools/p2p_probe.cu
// Run  :  build/p2p_probe [ndev] [bucket_mb] [grids e.g. 16,32,64,128]
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "CUDA %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); exit(1);} } while (0)

constexpr int kMaxDev = 8;
struct Ptrs { const char* p[kMaxDev]; };
struct WPtrs { char* p[kMaxDev]; };

__device__ __forceinline__ uint4 ld_na(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_plain(const void* p) {
  uint4 v;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_na(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float4 f4(const uint4& v) {
  return make_float4(__uint_as_float(v.x), __uint_as_float(v.y), __uint_as_float(v.z), __uint_as_float(v.w));
}

// ---------------------------------------------------------------- pull, register path
template <int W, int U, bool NA>
__global__ void __launch_bounds__(512, 1) pull_ldg(Ptrs src, uint64_t shard_off, uint64_t nvec, float* out, int self) {
  const uint64_t gstride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t v0 = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; v0 < nvec; v0 += gstride * U) {
    uint4 r[U][W];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint64_t v = v0 + u * gstride;
#pragma unroll
      for (int k = 0; k < W; ++k) {
        const int q = (self + k) % W;
        if (v < nvec) r[u][k] = NA ? ld_na(src.p[q] + shard_off + (v << 4)) : ld_plain(src.p[q] + shard_off + (v << 4));
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint64_t v = v0 + u * gstride;
      if (v < nvec) {
        float4 a = make_float4(0, 0, 0, 0);
#pragma unroll
        for (int k = 0; k < W; ++k) { float4 b = f4(r[u][k]); a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
        reinterpret_cast<float4*>(out)[v] = a;
      }
    }
  }
}

// ---------------------------------------------------------------- mbarrier / bulk-copy PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t parity) {
  // bounded: a protocol bug must trap, not hang the GPU
  for (uint32_t spins = 0; spins < (1u << 26); ++spins) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}" : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
    if (ok) return;
  }
  __trap();
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}

// ---------------------------------------------------------------- pull, TMA path
// warp 0 lane 0 = producer; warps 1..NC = consumers.  Stage = W chunks of CH bytes (one per peer).
template <int W, int CH, int S>
__global__ void __launch_bounds__(32 + 256, 1) pull_tma(Ptrs src, uint64_t shard_off, uint64_t nchunks, float* out, int self) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t full[S], empty[S];
  constexpr int NCW = 8;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], NCW); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp == 0) {
    if (lane == 0) {
      int s = 0; uint32_t ph = 0;
      for (uint64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
        mbar_wait(&empty[s], ph ^ 1);
        mbar_expect_tx(&full[s], W * CH);
#pragma unroll
        for (int k = 0; k < W; ++k) {
          const int q = (self + k) % W;
          bulk_g2s(smem + (size_t(s) * W + k) * CH, src.p[q] + shard_off + c * CH, CH, &full[s]);
        }
        if (++s == S) { s = 0; ph ^= 1; }
      }
    }
  } else {
    const int ct = threadIdx.x - 32;
    int s = 0; uint32_t ph = 0;
    for (uint64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
      mbar_wait(&full[s], ph);
      const unsigned char* st = smem + size_t(s) * W * CH;
#pragma unroll
      for (int v = ct; v < CH / 16; v += 256) {
        float4 a = make_float4(0, 0, 0, 0);
#pragma unroll
        for (int k = 0; k < W; ++k) {
          float4 b = *reinterpret_cast<const float4*>(st + size_t(k) * CH + (v << 4));
          a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
        }
        reinterpret_cast<float4*>(out)[c * (CH / 16) + v] = a;
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[s]);
      if (++s == S) { s = 0; ph ^= 1; }
    }
  }
}

// ---------------------------------------------------------------- push, register path
template <int W, int U>
__global__ void __launch_bounds__(512, 1) push_stg(WPtrs dst, uint64_t shard_off, uint64_t nvec, const float* in, int self) {
  const uint64_t gstride = uint64_t(gridDim.x) * blockDim.x;
  for (uint64_t v0 = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x; v0 < nvec; v0 += gstride * U) {
    uint4 r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { const uint64_t v = v0 + u * gstride; if (v < nvec) r[u] = reinterpret_cast<const uint4*>(in)[v]; }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint64_t v = v0 + u * gstride;
      if (v < nvec) {
#pragma unroll
        for (int k = 0; k < W; ++k) { const int q = (self + k) % W; st_na(dst.p[q] + shard_off + (v << 4), r[u]); }
      }
    }
  }
}

// ---------------------------------------------------------------- push, TMA path (one producer thread does everything)
template <int W, int CH, int S>
__global__ void __launch_bounds__(128, 1) push_tma(WPtrs dst, uint64_t shard_off, uint64_t nchunks, const float* in, int self) {
  extern __shared__ __align__(128) unsigned char smem[];
  __shared__ uint64_t full[S];
  if (threadIdx.x == 0) {
    for (int s = 0; s < S; ++s) mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // software pipeline: loads run S-1 chunks ahead of the stores
    uint64_t c_ld = blockIdx.x;
    int s_ld = 0; uint32_t ph = 0; int s_st = 0;
    int inflight = 0;
    uint64_t issued = 0, stored = 0;
    const uint64_t mine = (nchunks > blockIdx.x) ? (nchunks - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    while (stored < mine) {
      while (issued < mine && inflight < S) {
        // the slot's previous stores must have finished READING shared memory
        if (issued >= S) asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(S - 1) : "memory");
        mbar_expect_tx(&full[s_ld], CH);
        bulk_g2s(smem + size_t(s_ld) * CH, reinterpret_cast<const char*>(in) + c_ld * CH, CH, &full[s_ld]);
        c_ld += gridDim.x; ++issued; ++inflight;
        if (++s_ld == S) s_ld = 0;
      }
      mbar_wait(&full[s_st], ph);
      const uint64_t c = blockIdx.x + stored * gridDim.x;
#pragma unroll
      for (int k = 0; k < W; ++k) { const int q = (self + k) % W; bulk_s2g(dst.p[q] + shard_off + c * CH, smem + size_t(s_st) * CH, CH); }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      ++stored; --inflight;
      if (++s_st == S) { s_st = 0; ph ^= 1; }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

// ---------------------------------------------------------------- host
struct Dev {
  char* bucket = nullptr;   // N bytes
  float* shard = nullptr;   // N / ndev bytes
  cudaStream_t st;
  cudaEvent_t e0, e1;
};

int main(int argc, char** argv) {
  int ndev_avail = 0;
  CK(cudaGetDeviceCount(&ndev_avail));
  int ndev = argc > 1 ? atoi(argv[1]) : ndev_avail;
  if (ndev > ndev_avail) ndev = ndev_avail;
  if (ndev > kMaxDev) ndev = kMaxDev;
  const double mb = argc > 2 ? atof(argv[2]) : 64.0;
  std::vector<int> grids;
  { std::string g = argc > 3 ? argv[3] : "16,32,64,128"; size_t p = 0; while (p < g.size()) { grids.push_back(atoi(g.c_str() + p)); p = g.find(',', p); if (p == std::string::npos) break; ++p; } }
  const int iters = 10;
  const uint64_t quantum = uint64_t(ndev) * 65536;
  const uint64_t N = uint64_t(mb * 1048576.0) / quantum * quantum;
  const uint64_t shard_bytes = N / ndev;
  printf("# ndev %d  bucket %.1f MB  shard %.2f MB\n", ndev, N / 1048576.0, shard_bytes / 1048576.0);
  std::vector<Dev> D(ndev);
  for (int d = 0; d < ndev; ++d) {
    CK(cudaSetDevice(d));
    for (int q = 0; q < ndev; ++q) if (q != d) { cudaError_t e = cudaDeviceEnablePeerAccess(q, 0); if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CK(e); cudaGetLastError(); }
    CK(cudaMalloc(&D[d].bucket, N));
    CK(cudaMalloc(&D[d].shard, shard_bytes));
    CK(cudaMemset(D[d].bucket, 0, N));
    CK(cudaMemset(D[d].shard, 0, shard_bytes));
    CK(cudaStreamCreateWithFlags(&D[d].st, cudaStreamNonBlocking));
    CK(cudaEventCreate(&D[d].e0)); CK(cudaEventCreate(&D[d].e1));
  }
  Ptrs src; WPtrs dst;
  for (int q = 0; q < kMaxDev; ++q) { src.p[q] = q < ndev ? D[q].bucket : nullptr; dst.p[q] = q < ndev ? D[q].bucket : nullptr; }

  auto run = [&](const char* name, int grid, auto launch) {
    for (int rep = 0; rep < 2; ++rep) {          // rep 0 = warm-up
      for (int d = 0; d < ndev; ++d) { CK(cudaSetDevice(d)); CK(cudaDeviceSynchronize()); }
      for (int d = 0; d < ndev; ++d) {
        CK(cudaSetDevice(d));
        CK(cudaEventRecord(D[d].e0, D[d].st));
        for (int i = 0; i < (rep ? iters : 2); ++i) launch(d, grid);
        CK(cudaEventRecord(D[d].e1, D[d].st));
      }
      float worst = 0;
      for (int d = 0; d < ndev; ++d) {
        CK(cudaSetDevice(d)); CK(cudaStreamSynchronize(D[d].st)); CK(cudaGetLastError());
        float ms; CK(cudaEventElapsedTime(&ms, D[d].e0, D[d].e1)); if (ms > worst) worst = ms;
      }
      if (rep) {
        const double us = worst * 1e3 / iters;
        const double link = double(shard_bytes) * (ndev - 1);      // bytes crossing NVLink per device per launch
        printf("%-14s grid %3d  %8.1f us   %7.1f GB/s per direction\n", name, grid, us, link / us / 1e3);
        fflush(stdout);
      }
    }
  };

#define PULL_LDG(Wv, Uv, NAv) pull_ldg<Wv, Uv, NAv><<<grid, 512, 0, D[d].st>>>(src, uint64_t(d) * shard_bytes, shard_bytes / 16, D[d].shard, d)
#define PUSH_STG(Wv, Uv) push_stg<Wv, Uv><<<grid, 512, 0, D[d].st>>>(dst, uint64_t(d) * shard_bytes, shard_bytes / 16, D[d].shard, d)
  auto set_smem = [&](auto kern, int bytes) { for (int d = 0; d < ndev; ++d) { CK(cudaSetDevice(d)); CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes)); } };

  for (int grid : grids) {
    if (ndev == 2) {
      run("pull ldg_na", grid, [&](int d, int grid) { PULL_LDG(2, 8, true); });
      run("pull ldg", grid, [&](int d, int grid) { PULL_LDG(2, 8, false); });
      { constexpr int CH = 16384, S = 6; set_smem(pull_tma<2, CH, S>, 2 * CH * S);
        run("pull tma16k", grid, [&](int d, int grid) { pull_tma<2, CH, S><<<grid, 288, 2 * CH * S, D[d].st>>>(src, uint64_t(d) * shard_bytes, shard_bytes / CH, D[d].shard, d); }); }
      { constexpr int CH = 4096, S = 24; set_smem(pull_tma<2, CH, S>, 2 * CH * S);
        run("pull tma4k", grid, [&](int d, int grid) { pull_tma<2, CH, S><<<grid, 288, 2 * CH * S, D[d].st>>>(src, uint64_t(d) * shard_bytes, shard_bytes / CH, D[d].shard, d); }); }
      run("push stg_na", grid, [&](int d, int grid) { PUSH_STG(2, 8); });
      { constexpr int CH = 16384, S = 8; set_smem(push_tma<2, CH, S>, CH * S);
        run("push tma16k", grid, [&](int d, int grid) { push_tma<2, CH, S><<<grid, 128, CH * S, D[d].st>>>(dst, uint64_t(d) * shard_bytes, shard_bytes / CH, D[d].shard, d); }); }
    } else if (ndev == 4) {
      run("pull ldg_na", grid, [&](int d, int grid) { PULL_LDG(4, 4, true); });
      run("pull ldg", grid, [&](int d, int grid) { PULL_LDG(4, 4, false); });
      { constexpr int CH = 8192, S = 6; set_smem(pull_tma<4, CH, S>, 4 * CH * S);
        run("pull tma8k", grid, [&](int d, int grid) { pull_tma<4, CH, S><<<grid, 288, 4 * CH * S, D[d].st>>>(src, uint64_t(d) * shard_bytes, shard_bytes / CH, D[d].shard, d); }); }
      run("push stg_na", grid, [&](int d, int grid) { PUSH_STG(4, 4); });
      { constexpr int CH = 16384, S = 8; set_smem(push_tma<4, CH, S>, CH * S);
        run("push tma16k", grid, [&](int d, int grid) { push_tma<4, CH, S><<<grid, 128, CH * S, D[d].st>>>(dst, uint64_t(d) * shard_bytes, shard_bytes / CH, D[d].shard, d); }); }
    } else if (ndev == 8) {
      run("pull ldg_na", grid, [&](int d, int grid) { PULL_LDG(8, 2, true); });
      run("pull ldg", grid, [&](int d, int grid) { PULL_LDG(8, 2, false); });
      { constexpr int CH = 4096, S = 6; set_smem(pull_tma<8, CH, S>, 8 * CH * S);
        run("pull tma4k", grid, [&](int d, int grid) { pull_tma<8, CH, S><<<grid, 288, 8 * CH * S, D[d].st>>>(src, uint64_t(d) * shard_bytes, shard_bytes / CH, D[d].shard, d); }); }
      { constexpr int CH = 8192, S = 3; set_smem(pull_tma<8, CH, S>, 8 * CH * S);
        run("pull tma8k", grid, [&](int d, int grid) { pull_tma<8, CH, S><<<grid, 288, 8 * CH * S, D[d].st>>>(src, uint64_t(d) * shard_bytes, shard_bytes / CH, D[d].shard, d); }); }
      run("push stg_na", grid, [&](int d, int grid) { PUSH_STG(8, 4); });
      { constexpr int CH = 16384, S = 8; set_smem(push_tma<8, CH, S>, CH * S);
        run("push tma16k", grid, [&](int d, int grid) { push_tma<8, CH, S><<<grid, 128, CH * S, D[d].st>>>(dst, uint64_t(d) * shard_bytes, shard_bytes / CH, D[d].shard, d); }); }
    } else {
      fprintf(stderr, "ndev must be 2, 4 or 8\n");
      return 1;
    }
  }
  // reference: the copy engine, one direction, device 1 -> device 0
  {
    CK(cudaSetDevice(0));
    for (int rep = 0; rep < 2; ++rep) {
      CK(cudaEventRecord(D[0].e0, D[0].st));
      for (int i = 0; i < iters; ++i) CK(cudaMemcpyPeerAsync(D[0].bucket, 0, D[1].bucket, 1, N, D[0].st));
      CK(cudaEventRecord(D[0].e1, D[0].st));
      CK(cudaStreamSynchronize(D[0].st));
      float ms; CK(cudaEventElapsedTime(&ms, D[0].e0, D[0].e1));
      if (rep) printf("memcpyPeer 1->0 %8.1f us   %7.1f GB/s\n", ms * 1e3 / iters, double(N) / (ms * 1e3 / iters) / 1e3);
    }
  }
  return 0;
}
