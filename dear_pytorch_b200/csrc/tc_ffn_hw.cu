// tc_ffn_hw.cu — hand-written Hopper (sm_90a) wgmma GEMMs for the transformer FFN with the GELU in the epilogue.
//
//     ffn_up_hw    : H = gelu(Z),  Z = X W^T + b      X [M,K], W [N,K], b [N]  (bf16, fp32 accumulate)  ->  H, Z [M,N]
//     ffn_dgelu_hw : dZ = (dY Wt^T) * gelu'(Z)        dY [M,K], Wt [N,K] (= transposed down-projection weight), Z [M,N]
//   (one kernel template, two epilogue modes; A is K-major, B is K-major or MN-major)
//
// Why this kernel exists: a library GEMM followed by a GELU kernel writes the [tokens, 4*hidden] pre-activation, reads it
// back and writes the activation; here the epilogue applies bias + GELU (or GELU') to the accumulators before the one
// store, and the dgrad reads the down-projection weight as nn.Linear stores it.
//
// Structure (one CTA per SM, persistent over 128x128 output tiles, K step 64):
//   warpgroup 0     TMA producer (one thread): cp.async.bulk.tensor.2d (128B swizzle) A 128x64 + B 128x64 into a
//                   6-stage ring, mbarrier expect_tx / complete_tx.  It runs ahead into the next tile while the
//                   consumers are in their epilogue, so loads and the GELU math overlap.
//   warpgroups 1-2  consumers: each owns 64 rows of the tile and issues wgmma.mma_async m64n128k16 (bf16 in shared
//                   memory, fp32 accumulators in registers) x4 per stage; every warp releases the stage with one
//                   mbarrier arrive.  Epilogue straight from the accumulator registers: +bias -> erf-GELU -> bf16 stores.
// Every mbarrier wait is bounded and traps instead of spinning forever.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <torch/types.h>

#include <mutex>

namespace dear_tc {

void count_launch();

namespace hw {

constexpr int kTileM = 128, kTileN = 128, kTileK = 64, kWgmmaK = 16;
constexpr int kStages = 6;
constexpr int kABytes = kTileM * kTileK * 2;            // 16 KB
constexpr int kBBytes = kTileN * kTileK * 2;            // 16 KB
constexpr int kStageBytes = kABytes + kBBytes;          // 32 KB
constexpr int kNumThreads = 384;                        // 3 warpgroups: producer + 2 consumers
constexpr int kConsumerWarps = 8;
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /* alignment slack */ + 256 /* barriers */;
static_assert(kSmemBytes <= 227 * 1024, "shared memory ring exceeds the 227 KB a block may use");

// ---------------------------------------------------------------------------------------------- PTX
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `cta` of this cluster
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 remote;\n\t"
      "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [remote];\n\t}"
      ::"r"(smem_u32(bar)), "r"(cta)
      : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
// Bounded wait: a protocol bug must fail the launch (trap -> cudaErrorLaunchFailure), never wedge the GPU.
// try_wait itself suspends for an implementation-defined time, so the bound is wall time (2 s), not a spin count.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  while (!mbar_try_wait(bar, parity)) {
    if (global_timer_ns() - t0 > 2000000000ull) __trap();
  }
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
// the same box delivered into the shared memory (same CTA-relative offset) of every CTA in `mask`; each destination's
// mbarrier (same offset) receives the complete_tx
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma
__device__ __forceinline__ void fence_accumulators(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64x128, registers] += A[64x16, smem] * B[16x128, smem]; TRANS_B = 1: B is MN-major (n contiguous)
template <int TRANS_B>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
  asm volatile(
      "{\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "
      "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, "
      "%47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, 1, 1, 1, 0, %66;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
        "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),
        "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
        "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),
        "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
        "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
        "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),
        "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "n"(TRANS_B)
      : "memory");
}

// ------------------------------------------------------------------------------------- descriptors
// wgmma shared-memory matrix descriptor, 128-byte swizzle:
//   [0,14) start address >> 4   [16,30) leading byte offset >> 4   [32,46) stride byte offset >> 4
//   [49,52) base offset = 0 (tiles are 1024-byte aligned)   [62,64) layout type = 1 (SWIZZLE_128B)
// K-major operand: rows of 64 bf16 (128 bytes), SBO = 1024 B between 8-row groups, LBO unused.
// MN-major operand (B[n][k] = W[k][n] for a row-major W [K, N]): canonical layout in 16-byte units
// ((8,n),(8,k)) : ((1,LBO),(8,SBO)) — an atom is 8 k-rows of 128 bytes (64 contiguous n); LBO = distance between 64-wide
// n blocks, SBO = distance between 8-row k groups.  A stage holds kTileN/64 blocks of {64 n, kTileK k} = 8 KB each, so
// LBO = 8192 B and SBO = 1024 B.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(lbo >> 4) << 16;
  d |= static_cast<uint64_t>(1024 >> 4) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// ------------------------------------------------------------------------------------------ GELU
// Phi(-|x|) by Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7): 2 MUFU + ~12 FMA per element
__device__ __forceinline__ float gelu_fast(float x) {
  const float ax = fabsf(x);
  const float e = __expf(-0.5f * x * x);
  const float t = __fdividef(1.0f, fmaf(0.3275911f * 0.70710678118654752440f, ax, 1.0f));
  float p = 1.061405429f;
  p = fmaf(p, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float q = 0.5f * p * t * e;
  return x * (x < 0.f ? q : 1.0f - q);
}

// d/dz [z Phi(z)] = Phi(z) + z phi(z); phi shares exp(-z^2/2) with the tail
__device__ __forceinline__ float dgelu_fast(float z) {
  const float az = fabsf(z);
  const float e = __expf(-0.5f * z * z);
  const float t = __fdividef(1.0f, fmaf(0.3275911f * 0.70710678118654752440f, az, 1.0f));
  float p = 1.061405429f;
  p = fmaf(p, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float q = 0.5f * p * t * e;
  return fmaf(z, 0.39894228040143267794f * e, z < 0.f ? q : 1.0f - q);
}

__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// -------------------------------------------------------------------------------------------- kernel
// MODE_UP   : aux = bias [N];      out0 = H = gelu(acc + bias), out1 = Z = acc + bias
// MODE_DGELU: aux = Z [M,N] (read); out0 = dZ = acc * gelu'(Z),  out1 unused
enum EpilogueMode { MODE_UP = 0, MODE_DGELU = 1 };

// B operand of the MN-major path split into pieces of {64 n, kPieceK k}: enough pieces that every CTA of a cluster
// loads (and multicasts) the same number
template <int CL>
struct BmnPieces {
  static constexpr int kNBlocks = kTileN / 64;
  static constexpr int kCount = kNBlocks > CL ? kNBlocks : CL;
  static constexpr int kPerBlock = kCount / kNBlocks;
  static constexpr int kRowsK = kTileK / kPerBlock;
};

// BMN: the B operand is given as a row-major [K, N] matrix (MN-major) instead of [N, K] (K-major): the dgrad GEMM
// dH = dY W2 reads the nn.Linear weight W2 [hidden, inter] as it is stored — no transposed copy per step.
// CL: CTAs per cluster (1, 2 or 4).  The CTAs of a cluster work on vertically adjacent output tiles (same n range); each
// loads 1/CL of the B tile and MULTICASTS it to all of them, so per K step a CTA makes L2 serve 16 + 16/CL KB instead of
// 32 KB.
template <int MODE, bool BMN, int CL>
__global__ void __launch_bounds__(kNumThreads, 1)
ffn_hw_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
              const __nv_bfloat16* __restrict__ aux, __nv_bfloat16* __restrict__ out0, __nv_bfloat16* __restrict__ out1,
              int M, int N, int K) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* full_bar = bars;                             // [kStages]   TMA -> consumers
  uint64_t* empty_bar = bars + kStages;                  // [kStages]   consumers (of every CTA in the cluster) -> TMA

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int tiles_m = (M + kTileM - 1) / kTileM, tiles_n = (N + kTileN - 1) / kTileN;
  const int num_kb = (K + kTileK - 1) / kTileK;
  // cluster-tile schedule: cluster c takes every (gridDim/CL)-th group of CL vertically adjacent tiles
  const int crank = (CL > 1) ? static_cast<int>(cluster_ctarank()) : 0;
  const int cid = blockIdx.x / CL, ncl = gridDim.x / CL;
  const int tiles_mc = tiles_m / CL;                     // the host guarantees tiles_m % CL == 0
  const int num_ct = tiles_mc * tiles_n;
  constexpr uint16_t kAllCtas = static_cast<uint16_t>((1u << CL) - 1);

  if (threadIdx.x == 0) {
    prefetch_tmap(&tmap_a);
    prefetch_tmap(&tmap_b);
    for (int s = 0; s < kStages; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], kConsumerWarps * CL); }
    fence_barrier_init();
  }
  __syncthreads();
  if (CL > 1) cluster_sync_all();                        // the peers' barriers exist before anything signals them

  if (wg == 0) {
    // ===================================================================== TMA producer (one thread)
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int ct = cid; ct < num_ct; ct += ncl) {
        const int m0 = ((ct % tiles_mc) * CL + crank) * kTileM, n0 = (ct / tiles_mc) * kTileN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);                     // slot free in EVERY CTA of the cluster
          mbar_expect_tx(&full_bar[stage], kStageBytes);               // OOB rows/columns are zero-filled AND counted
          uint8_t* a_dst = smem + stage * kStageBytes;
          tma_load_2d(a_dst, &tmap_a, &full_bar[stage], kb * kTileK, m0);
          if (BMN) {
            // pieces of {64 n (contiguous), kRowsK k}, 128B-swizzled by the k row; block j of 64 n at j * 8 KB
            using P = BmnPieces<CL>;
#pragma unroll
            for (int j = 0; j < P::kCount / CL; ++j) {
              const int p = crank * (P::kCount / CL) + j, nb = p / P::kPerBlock, kp = p % P::kPerBlock;
              uint8_t* dst = a_dst + kABytes + nb * (kTileK * 128) + kp * (P::kRowsK * 128);
              if (CL > 1) tma_load_2d_mc(dst, &tmap_b, &full_bar[stage], n0 + nb * 64, kb * kTileK + kp * P::kRowsK, kAllCtas);
              else tma_load_2d(dst, &tmap_b, &full_bar[stage], n0 + nb * 64, kb * kTileK + kp * P::kRowsK);
            }
          } else if (CL > 1) {
            // rows [n0 + crank*kTileN/CL, +kTileN/CL) of B, delivered to every CTA (the map's box has kTileN / CL rows)
            tma_load_2d_mc(a_dst + kABytes + crank * (kBBytes / CL), &tmap_b, &full_bar[stage], kb * kTileK,
                           n0 + crank * (kTileN / CL), kAllCtas);
          } else {
            tma_load_2d(a_dst + kABytes, &tmap_b, &full_bar[stage], kb * kTileK, n0);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ============================================================ consumers: 2 warpgroups x 64 rows
    const int cw = wg - 1;                                             // rows cw*64 .. cw*64+63 of the tile
    const int wq = warp & 3;                                           // warp within the warpgroup: 16 rows each
    int stage = 0; uint32_t phase = 0;
    for (int ct = cid; ct < num_ct; ct += ncl) {
      const int m0 = ((ct % tiles_mc) * CL + crank) * kTileM, n0 = (ct / tiles_mc) * kTileN;
      float d[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) d[i] = 0.f;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);                            // TMA bytes have landed
        const uint32_t a_addr = smem_u32(smem + stage * kStageBytes) + cw * (64 * 128);
        const uint32_t b_addr = smem_u32(smem + stage * kStageBytes + kABytes);
        fence_accumulators(d);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kTileK / kWgmmaK; ++k) {
          // K advance: K-major operands move +32 bytes inside the 128-byte swizzle row per 16 bf16; the MN-major
          // operand moves two 8-row k groups (2 x 1024 bytes)
          const uint64_t adesc = make_smem_desc(a_addr + k * kWgmmaK * 2, 16);
          if (BMN) wgmma_m64n128k16<1>(d, adesc, make_smem_desc(b_addr + k * (kWgmmaK / 8) * 1024, kTileK * 128));
          else wgmma_m64n128k16<0>(d, adesc, make_smem_desc(b_addr + k * kWgmmaK * 2, 16));
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_accumulators(d);
        // this warp's reads of the stage are complete: release it in every CTA whose multicast load refills it
        if (CL > 1) { if (lane < CL) mbar_arrive_cluster(&empty_bar[stage], lane); }
        else if (lane == 0) mbar_arrive(&empty_bar[stage]);
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }

      // epilogue: accumulator d[4i + {0,1}] is (row r, cols 8i + 2(lane%4) + {0,1}), d[4i + {2,3}] is row r + 8
      const int r0 = m0 + cw * 64 + wq * 16 + (lane >> 2);
      const int cbase = n0 + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < kTileN / 8; ++i) {
        const int col = cbase + 8 * i;
        if (col >= N) continue;                                        // N % 8 == 0: a column pair is all-in or all-out
        if (MODE == MODE_UP) {
          const uint32_t bw = __ldg(reinterpret_cast<const unsigned int*>(aux + col));
          const float b0 = __uint_as_float(bw << 16), b1 = __uint_as_float(bw & 0xffff0000u);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            if (row < M) {
              const float z0 = d[4 * i + 2 * h] + b0, z1 = d[4 * i + 2 * h + 1] + b1;
              const size_t off = static_cast<size_t>(row) * N + col;
              *reinterpret_cast<uint32_t*>(out1 + off) = pack_bf16(z0, z1);
              *reinterpret_cast<uint32_t*>(out0 + off) = pack_bf16(gelu_fast(z0), gelu_fast(z1));
            }
          }
        } else {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int row = r0 + 8 * h;
            if (row < M) {
              const size_t off = static_cast<size_t>(row) * N + col;
              const uint32_t zw = __ldg(reinterpret_cast<const unsigned int*>(aux + off));
              const float z0 = __uint_as_float(zw << 16), z1 = __uint_as_float(zw & 0xffff0000u);
              *reinterpret_cast<uint32_t*>(out0 + off) =
                  pack_bf16(d[4 * i + 2 * h] * dgelu_fast(z0), d[4 * i + 2 * h + 1] * dgelu_fast(z1));
            }
          }
        }
      }
    }
  }

  // ------------------------------------------------------------------------------------- teardown
  __syncthreads();
  if (CL > 1) cluster_sync_all();                        // no multicast / remote arrive may target a CTA that has exited
}

// -------------------------------------------------------------------------------------------- host
using EncodeTiledFn = PFN_cuTensorMapEncodeTiled_v12000;

static EncodeTiledFn encode_tiled() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    auto err = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    TORCH_CHECK(err == cudaSuccess && q == cudaDriverEntryPointSuccess && p != nullptr, "cuTensorMapEncodeTiled is not available");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// 2-D row-major bf16 matrix [rows, cols]; box = box_rows x box_cols (box_cols = 64: 128 bytes = one swizzle row)
static CUtensorMap make_tmap(const void* base, int64_t rows, int64_t cols, int box_rows, int box_cols) {
  CUtensorMap m;
  const cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  const cuuint64_t gstride[1] = {static_cast<cuuint64_t>(cols) * 2};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(box_cols), static_cast<cuuint32_t>(box_rows)};
  const cuuint32_t estr[2] = {1, 1};
  CUresult r = encode_tiled()(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                              CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  TORCH_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with code ", static_cast<int>(r));
  return m;
}

}  // namespace hw

static void check_bf16(const at::Tensor& t, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16 && t.is_contiguous() &&
              reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0, what, ": contiguous 16-byte aligned CUDA bf16 tensor expected");
}

template <int MODE, bool BMN, int CL>
static void launch_hw_cl(const at::Tensor& a, const at::Tensor& b, const __nv_bfloat16* aux, at::Tensor& out0, at::Tensor* out1,
                         int M, int N, int K) {
  const CUtensorMap ta = hw::make_tmap(a.data_ptr(), M, K, hw::kTileM, hw::kTileK);
  // MN-major B: row-major [K, N] read in pieces of 64 columns (128 bytes) x kRowsK rows
  const CUtensorMap tb = BMN ? hw::make_tmap(b.data_ptr(), K, N, hw::BmnPieces<CL>::kRowsK, 64)
                             : hw::make_tmap(b.data_ptr(), N, K, hw::kTileN / CL, hw::kTileK);
  static std::once_flag attr_once;
  std::call_once(attr_once, [] {
    C10_CUDA_CHECK(cudaFuncSetAttribute(hw::ffn_hw_kernel<MODE, BMN, CL>, cudaFuncAttributeMaxDynamicSharedMemorySize, hw::kSmemBytes));
  });
  const int tiles = ((M + hw::kTileM - 1) / hw::kTileM) * ((N + hw::kTileN - 1) / hw::kTileN);
  const int sms = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  auto stream = at::cuda::getCurrentCUDAStream().stream();
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(std::max(CL, sms / CL * CL));
  cfg.blockDim = dim3(hw::kNumThreads);
  cfg.dynamicSmemBytes = hw::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CL;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  // persistent kernel: one resident cluster per slot the hardware can co-schedule (GPC boundaries strand a few SMs
  // for clusters of 4), never more than there are cluster-tiles
  static int max_clusters = 0;
  if (max_clusters == 0) {
    int n = 0;
    if (CL == 1 || cudaOccupancyMaxActiveClusters(&n, hw::ffn_hw_kernel<MODE, BMN, CL>, &cfg) != cudaSuccess || n <= 0) {
      cudaGetLastError();
      n = sms / CL;
    }
    max_clusters = n;
  }
  const int grid = std::max(1, std::min(tiles / CL, max_clusters)) * CL;
  cfg.gridDim = dim3(grid);
  C10_CUDA_CHECK(cudaLaunchKernelEx(&cfg, hw::ffn_hw_kernel<MODE, BMN, CL>, ta, tb, aux,
                                    reinterpret_cast<__nv_bfloat16*>(out0.data_ptr()),
                                    out1 != nullptr ? reinterpret_cast<__nv_bfloat16*>(out1->data_ptr()) : nullptr, M, N, K));
  count_launch();
}

static int g_force_cluster = -1;       // -1: default (1 CTA per cluster); 1 / 2 / 4: forced (benchmarks, tests)
void set_ffn_hw_cluster(int cl) { g_force_cluster = cl; }

template <int MODE, bool BMN = false>
static void launch_hw(const at::Tensor& a, const at::Tensor& b, const __nv_bfloat16* aux, at::Tensor& out0, at::Tensor* out1,
                      int M, int N, int K) {
  const int tiles_m = (M + hw::kTileM - 1) / hw::kTileM;
  // the CTAs of a cluster take vertically adjacent tiles: the cluster size must divide the number of tile rows
  int cl = g_force_cluster > 0 ? g_force_cluster : 1;
  while (cl > 1 && tiles_m % cl != 0) cl >>= 1;
  if (cl >= 4) launch_hw_cl<MODE, BMN, 4>(a, b, aux, out0, out1, M, N, K);
  else if (cl == 2) launch_hw_cl<MODE, BMN, 2>(a, b, aux, out0, out1, M, N, K);
  else launch_hw_cl<MODE, BMN, 1>(a, b, aux, out0, out1, M, N, K);
}

// H, Z = gelu(X W^T + b), X W^T + b
std::vector<at::Tensor> ffn_up_hw(const at::Tensor& x, const at::Tensor& w, const at::Tensor& bias) {
  check_bf16(x, "ffn_up_hw x"); check_bf16(w, "ffn_up_hw w"); check_bf16(bias, "ffn_up_hw bias");
  TORCH_CHECK(x.dim() == 2 && w.dim() == 2 && x.size(1) == w.size(1) && bias.numel() == w.size(0), "ffn_up_hw: shape mismatch");
  const int M = x.size(0), K = x.size(1), N = w.size(0);
  TORCH_CHECK(K % 8 == 0 && N % 8 == 0, "ffn_up_hw: K and N must be multiples of 8");
  c10::cuda::CUDAGuard guard(x.device());
  auto h = at::empty({M, N}, x.options());
  auto z = at::empty({M, N}, x.options());
  if (M == 0) return {h, z};
  launch_hw<hw::MODE_UP>(x, w, reinterpret_cast<const __nv_bfloat16*>(bias.data_ptr()), h, &z, M, N, K);
  return {h, z};
}

// dZ = (dY Wt^T) * gelu'(Z)   with   Wt = W^T stored [N, K] row-major (K-major operand: the caller keeps a transposed
// copy of the down-projection weight W [K, N])
at::Tensor ffn_dgelu_hw(const at::Tensor& dy, const at::Tensor& wt, const at::Tensor& z) {
  check_bf16(dy, "ffn_dgelu_hw dy"); check_bf16(wt, "ffn_dgelu_hw wt"); check_bf16(z, "ffn_dgelu_hw z");
  TORCH_CHECK(dy.dim() == 2 && wt.dim() == 2 && z.dim() == 2 && dy.size(1) == wt.size(1) && z.size(0) == dy.size(0) &&
              z.size(1) == wt.size(0), "ffn_dgelu_hw: shape mismatch (dy [M,K], wt [N,K], z [M,N])");
  const int M = dy.size(0), K = dy.size(1), N = wt.size(0);
  TORCH_CHECK(K % 8 == 0 && N % 8 == 0, "ffn_dgelu_hw: K and N must be multiples of 8");
  c10::cuda::CUDAGuard guard(dy.device());
  auto dz = at::empty({M, N}, dy.options());
  if (M == 0) return dz;
  launch_hw<hw::MODE_DGELU>(dy, wt, reinterpret_cast<const __nv_bfloat16*>(z.data_ptr()), dz, nullptr, M, N, K);
  return dz;
}

// dZ = (dY W) * gelu'(Z)   with the nn.Linear weight W [K, N] = [hidden, inter] exactly as it is stored (MN-major B
// operand): the dgrad of the down projection fused with the GELU backward, no transposed copy of W.
at::Tensor ffn_dgelu_hw_nt(const at::Tensor& dy, const at::Tensor& w, const at::Tensor& z) {
  check_bf16(dy, "ffn_dgelu_hw_nt dy"); check_bf16(w, "ffn_dgelu_hw_nt w"); check_bf16(z, "ffn_dgelu_hw_nt z");
  TORCH_CHECK(dy.dim() == 2 && w.dim() == 2 && z.dim() == 2 && dy.size(1) == w.size(0) && z.size(0) == dy.size(0) &&
              z.size(1) == w.size(1), "ffn_dgelu_hw_nt: shape mismatch (dy [M,K], w [K,N], z [M,N])");
  const int M = dy.size(0), K = dy.size(1), N = w.size(1);
  TORCH_CHECK(K % 8 == 0 && N % 8 == 0, "ffn_dgelu_hw_nt: K and N must be multiples of 8");
  c10::cuda::CUDAGuard guard(dy.device());
  auto dz = at::empty({M, N}, dy.options());
  if (M == 0) return dz;
  launch_hw<hw::MODE_DGELU, true>(dy, w, reinterpret_cast<const __nv_bfloat16*>(z.data_ptr()), dz, nullptr, M, N, K);
  return dz;
}

}  // namespace dear_tc
