// rs_pipe.cu — Kernel A, stripe-pipelined variant (sm_90a): gradient pack + reduce-scatter + fp32
// accumulate + 1/P scale for buckets that are bandwidth-bound (>= a few MB).
//
// Replaces, like the one-shot rs_kernel in kernels.cu: the per-parameter bucket copy_
// (dear/dear_dopt.py:265), ncclReduceScatter (common/comm_core/src/communicator.cpp:157-169) and div_ (:306).
//
// Why a second variant.  The one-shot kernel packs the WHOLE bucket, crosses one flag round and then pulls:
// for a large bucket the pack is a large fraction of the kernel — NVLink idles while HBM copies and vice versa.  Here the shard is cut into stripes; stripe k of every shard is packed
// and published while stripe k-1 is being pulled, and the pull itself is moved off the LSU:
//
//   warps 7-18  PACK      copy this rank's gradients into the symmetric bucket, stripe-major, from a host-built work
//                         list of <= 32 KB copies (BucketSet::set_pack); the CTA that completes stripe k grid-wide
//                         publishes RS_READY = (epoch<<8 | k+1) to all peers
//   warp  0     PRODUCER  one lane: wait for every peer's stripe-k flag, then feed a 12 x 16 KB shared-memory
//                         ring with cp.async.bulk (UBLKCP) copies straight out of the PEERS' buckets over NVLink;
//                         one ring slot = one 16 KB chunk of my shard from one peer, mbarrier complete_tx
//   warps 1-6   REDUCE    accumulate the P slots of a chunk in fp32 registers (fixed peer order => run-to-run
//                         deterministic), scale by 1/P, write the fp32 shard
//
// Bulk-copy pulls (tools/p2p_probe.cu compares them with 128-bit register loads) need fewer CTAs to keep NVLink busy,
// and they leave the CTA's threads free to run the pack concurrently.
#include <cuda_runtime.h>
#include <stdexcept>
#include <string>
#include "dear_common.h"
#include "dear_device.cuh"

namespace dear {

constexpr int kPipeStages = 12;                         // 12 x 16 KB = 192 KB ring per CTA
constexpr int kReduceThreads = 192;
constexpr int kPackThreads = 384;
constexpr int kPipeThreads = 32 + kReduceThreads + kPackThreads;  // 608
constexpr int kPackVecs = (kPipePackPiece / 16 + kPackThreads - 1) / kPackThreads;     // 6 x 128-bit per pack thread per piece
constexpr int kRedVecs = (kPipeChunk / 16 + kReduceThreads - 1) / kReduceThreads;      // 6 x 128-bit per reduce thread per chunk

// ---- mbarrier / bulk-copy PTX ----------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(b)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* b, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(b)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Wait for a phase, but give up when the CTA-wide abort word is raised (a cross-GPU wait timed out somewhere):
// a protocol failure must end in an error on the host, never in a hung GPU.
__device__ __forceinline__ bool mbar_wait(uint64_t* b, uint32_t parity, const volatile uint32_t* abort_word) {
  uint32_t spins = 0;
  while (!mbar_try_wait(b, parity)) {
    if (((++spins) & 0xff) == 0 && *abort_word) return false;
  }
  return true;
}
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// One entry of the host-built work list: copy (or zero-fill) `nbytes` <= kPipePackPiece bytes into the bucket.
// All loads first (6 x 128 bit in flight per thread, 384 threads => 36 KB in flight per CTA), then the stores.
__device__ __forceinline__ void pack_piece(const PackSeg& pc, char* bucket, int ptid) {
  char* d = bucket + pc.dst_off;
  const uint32_t nb = uint32_t(pc.nbytes);
  const uint32_t nvec = nb >> 4;
  if (pc.flags & SEG_ZERO_FILL) {
    const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
    for (int j = 0; j < kPackVecs; ++j) {
      const uint32_t v = ptid + j * kPackThreads;
      if (v < nvec) st_stream(d + (size_t(v) << 4), z);
    }
    for (uint32_t b = (nvec << 4) + ptid * 2; b < nb; b += kPackThreads * 2) *reinterpret_cast<uint16_t*>(d + b) = 0;
    return;
  }
  const char* s = reinterpret_cast<const char*>(pc.src);
  uint4 r[kPackVecs];
#pragma unroll
  for (int j = 0; j < kPackVecs; ++j) {
    const uint32_t v = ptid + j * kPackThreads;
    if (v < nvec) r[j] = ld_stream(s + (size_t(v) << 4));
  }
#pragma unroll
  for (int j = 0; j < kPackVecs; ++j) {
    const uint32_t v = ptid + j * kPackThreads;
    if (v < nvec) st_stream(d + (size_t(v) << 4), r[j]);
  }
  for (uint32_t b = (nvec << 4) + ptid * 2; b < nb; b += kPackThreads * 2)
    *reinterpret_cast<uint16_t*>(d + b) = *reinterpret_cast<const uint16_t*>(s + b);
}

// The chunks of all stripes form one sequence that is dealt round-robin over the CTAs: the first chunk of stripe k
// that belongs to this CTA (every stripe but the last holds stripe_bytes / kPipeChunk chunks).
__device__ __forceinline__ uint32_t first_chunk(uint32_t k, uint64_t stripe_bytes) {
  const uint32_t before = uint32_t((uint64_t(k) * (stripe_bytes / kPipeChunk)) % gridDim.x);
  return (blockIdx.x + gridDim.x - before) % gridDim.x;
}

// AMP: dynamic loss scaling (p.amp != nullptr), CLIP: global-norm clipping (p.clip != nullptr), see rs_kernel in kernels.cu.
template <typename T, bool AMP, bool CLIP>
__global__ void __launch_bounds__(kPipeThreads, 1) rs_pipe_kernel(const RSParams p) {
  using Tr = ElemTraits<T>;
  constexpr int EV = Tr::kPerVec;
  extern __shared__ __align__(128) unsigned char ring[];          // kPipeStages x kPipeChunk
  __shared__ uint64_t s_full[kPipeStages], s_empty[kPipeStages];
  __shared__ uint32_t s_abort, s_last;

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const int world = p.world;
  void* sig_local = p.sig.ptr[p.rank];
  const uint32_t ch_ready = bucket_channel(p.bucket, RS_READY);
  const uint32_t ch_done = bucket_channel(p.bucket, RS_DONE);
  uint32_t* epoch_p = p.ctrl + ch_ready;
  uint32_t* cnt_pack = p.ctrl + kNumChannels + ch_ready;
  uint32_t* cnt_exit = p.ctrl + kNumChannels + ch_done;
  const uint32_t e = *reinterpret_cast<volatile uint32_t*>(epoch_p) + 1;
  const uint32_t e8 = e << 8;

  // (0) my bucket may still be read by a peer's previous reduce-scatter.
  wait_all_peers(sig_local, ch_done, e - 1, world, p.timeout_ns, p.status, ST_TIMEOUT_RS_DONE);

  const bool packing = p.pieces != nullptr;
  if (tid == 0) {
    for (int s = 0; s < kPipeStages; ++s) {
      mbar_init(&s_full[s], 1);
      mbar_init(&s_empty[s], kReduceThreads / 32);
    }
    s_abort = 0;
    s_last = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const volatile uint32_t* abort_word = &s_abort;

  const uint64_t SB = p.shard_elems * sizeof(T);         // bytes per shard
  const uint32_t K = p.nstripes;
  const uint64_t cs = p.stripe_bytes;
  const uint64_t my_shard_off = uint64_t(p.rank) * SB;
  bool bad = false;                               // AMP: this thread wrote a non-finite value
  float ss = 0.f;                                 // CLIP: sum of squares of the values this thread wrote

  if (tid >= 32 + kReduceThreads) {
    // ================================ PACK ================================
    const int ptid = tid - (32 + kReduceThreads);
    char* bucket = reinterpret_cast<char*>(p.grad.ptr[p.rank]);
    for (uint32_t k = 0; k < K; ++k) {
      if (packing) {
        // stripe k's work items, dealt round-robin over the CTAs (rotated per stripe so nobody is always first)
        const uint32_t lo = p.piece_first[k], hi = p.piece_first[k + 1];
        for (uint32_t i = lo + (blockIdx.x + gridDim.x - (lo % gridDim.x)) % gridDim.x; i < hi; i += gridDim.x) {
          PackSeg pc;
          const uint4* raw = reinterpret_cast<const uint4*>(p.pieces + i);
          const uint4 a = __ldg(raw), b2 = __ldg(raw + 1);
          pc.src = reinterpret_cast<const void*>(uint64_t(a.x) | (uint64_t(a.y) << 32));
          pc.dst_off = uint64_t(a.z) | (uint64_t(a.w) << 32);
          pc.nbytes = uint64_t(b2.x) | (uint64_t(b2.y) << 32);
          pc.tile_begin = b2.z;
          pc.flags = b2.w;
          pack_piece(pc, bucket, ptid);
        }
      }
      // stripe k is packed on this CTA; the CTA that completes it grid-wide publishes it to every peer
      named_bar_sync(1, kPackThreads);
      if (ptid == 0) {
        __threadfence();
        const uint32_t old = atomicAdd(cnt_pack, 1u);
        __threadfence();
        s_last = (old == gridDim.x * (k + 1) - 1) ? 1u : 0u;
      }
      named_bar_sync(1, kPackThreads);
      if (s_last != 0 && ptid < world) {
        __threadfence_system();
        st_release_sys(flag_at(p.sig.ptr[ptid], ch_ready, p.rank), e8 | (k + 1));
      }
    }
  } else if (tid < 32) {
    // ============================== PRODUCER ==============================
    if (lane == 0) {
      int s = 0;
      uint32_t ph = 0;
      bool ok = true;
      for (uint32_t k = 0; k < K && ok; ++k) {
        const uint64_t s_lo = uint64_t(k) * cs;
        if (s_lo >= SB) break;
        for (int q = 0; q < world && ok; ++q)
          ok = wait_flag(flag_at(sig_local, ch_ready, q), e8 | (k + 1), p.timeout_ns, p.status, ST_TIMEOUT_RS_READY);
        if (!ok) break;
        // the peers' data was written through the generic proxy; the bulk copies read it through the async proxy
        asm volatile("fence.proxy.async;" ::: "memory");
        const uint64_t s_hi = (s_lo + cs < SB) ? s_lo + cs : SB;
        const uint32_t nch = uint32_t((s_hi - s_lo + kPipeChunk - 1) / kPipeChunk);
        for (uint32_t c = first_chunk(k, cs); c < nch && ok; c += gridDim.x) {
          const uint64_t off = s_lo + uint64_t(c) * kPipeChunk;
          const uint32_t bytes = (off + kPipeChunk <= s_hi) ? kPipeChunk : uint32_t(s_hi - off);
          for (int j = 0; j < world; ++j) {
            const int q = (p.rank + 1 + j) % world;       // peers first, my own bucket last
            if (!mbar_wait(&s_empty[s], ph ^ 1, abort_word)) { ok = false; break; }
            mbar_expect_tx(&s_full[s], bytes);
            bulk_g2s(ring + size_t(s) * kPipeChunk, reinterpret_cast<const char*>(p.grad.ptr[q]) + my_shard_off + off, bytes,
                     &s_full[s]);
            if (++s == kPipeStages) { s = 0; ph ^= 1; }
          }
        }
      }
      if (!ok) *reinterpret_cast<volatile uint32_t*>(&s_abort) = 1u;
    }
  } else {
    // =============================== REDUCE ===============================
    const int rtid = tid - 32;
    const float scale = AMP ? p.scale * (1.f / *reinterpret_cast<volatile float*>(&p.amp->scale)) : p.scale;
    int s = 0;
    uint32_t ph = 0;
    bool ok = true;
    for (uint32_t k = 0; k < K && ok; ++k) {
      const uint64_t s_lo = uint64_t(k) * cs;
      if (s_lo >= SB) break;
      const uint64_t s_hi = (s_lo + cs < SB) ? s_lo + cs : SB;
      const uint32_t nch = uint32_t((s_hi - s_lo + kPipeChunk - 1) / kPipeChunk);
      for (uint32_t c = first_chunk(k, cs); c < nch && ok; c += gridDim.x) {
        const uint64_t off = s_lo + uint64_t(c) * kPipeChunk;
        const uint32_t bytes = (off + kPipeChunk <= s_hi) ? kPipeChunk : uint32_t(s_hi - off);
        const uint32_t nvec = bytes >> 4;
        float acc[kRedVecs][EV];
#pragma unroll
        for (int i = 0; i < kRedVecs; ++i)
#pragma unroll
          for (int x = 0; x < EV; ++x) acc[i][x] = 0.f;
        for (int j = 0; j < world; ++j) {
          // warp-uniform outcome: a lane that gave up must not leave its warp mates at the __syncwarp below
          if (!__all_sync(0xffffffffu, mbar_wait(&s_full[s], ph, abort_word))) { ok = false; break; }
          const unsigned char* st = ring + size_t(s) * kPipeChunk;
#pragma unroll
          for (int i = 0; i < kRedVecs; ++i) {
            const uint32_t v = rtid + i * kReduceThreads;
            if (v < nvec) {
              float f[EV];
              Tr::unpack(*reinterpret_cast<const uint4*>(st + (size_t(v) << 4)), f);
#pragma unroll
              for (int x = 0; x < EV; ++x) acc[i][x] += f[x];
            }
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&s_empty[s]);
          if (++s == kPipeStages) { s = 0; ph ^= 1; }
        }
        if (!ok) break;
        float* out = p.out + off / sizeof(T);
#pragma unroll
        for (int i = 0; i < kRedVecs; ++i) {
          const uint32_t v = rtid + i * kReduceThreads;
          if (v < nvec) {
#pragma unroll
            for (int x = 0; x < EV; ++x) acc[i][x] *= scale;
            if (AMP) bad |= !all_finite<EV>(acc[i]);
            if (CLIP) ss += sum_sq<EV>(acc[i]);
            float4* o = reinterpret_cast<float4*>(out + size_t(v) * EV);
            o[0] = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
            if (EV == 8) o[1] = make_float4(acc[i][EV - 4], acc[i][EV - 3], acc[i][EV - 2], acc[i][EV - 1]);
          }
        }
      }
    }
  }

  // AMP: one atomic per CTA into this rank's overflow word (every role reaches this point)
  if (AMP) {
    if (__syncthreads_or(bad) && tid == 0) atomicOr(&p.amp->overflow, 1u);
  }
  if (CLIP) clip_store_cta_partial(p.clip, p.clip_slot, ss);

  // (end) tell every peer I am done reading its bucket; advance the epoch.
  if (grid_arrive_is_last(cnt_exit)) {
    signal_all_peers(p.sig, ch_done, p.rank, world, e);
    if (tid == 0) {
      if (CLIP) clip_combine_slot(p.clip, p.clip_slot);
      *cnt_exit = 0;
      *cnt_pack = 0;
      *epoch_p = e;
    }
  }
}

static bool g_pipe_attr_set[12] = {false};

template <typename T, bool AMP, bool CLIP>
static void launch_pipe_ta(const RSParams& p, int grid, cudaStream_t s, int slot) {
  constexpr int smem = kPipeStages * kPipeChunk;
  if (!g_pipe_attr_set[slot]) {
    cudaError_t err = cudaFuncSetAttribute(rs_pipe_kernel<T, AMP, CLIP>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (err != cudaSuccess)
      throw std::runtime_error(std::string("dear: cannot reserve shared memory for rs_pipe_kernel: ") + cudaGetErrorString(err));
    g_pipe_attr_set[slot] = true;
  }
  rs_pipe_kernel<T, AMP, CLIP><<<grid, kPipeThreads, smem, s>>>(p);
}

template <typename T>
static void launch_pipe_t(const RSParams& p, int grid, cudaStream_t s, int slot) {
  const bool clip = p.clip != nullptr;
  if (p.amp != nullptr) clip ? launch_pipe_ta<T, true, true>(p, grid, s, 9 + slot) : launch_pipe_ta<T, true, false>(p, grid, s, 3 + slot);
  else clip ? launch_pipe_ta<T, false, true>(p, grid, s, 6 + slot) : launch_pipe_ta<T, false, false>(p, grid, s, slot);
}

void launch_rs_pipe(const RSParams& p, int grid, cudaStream_t s) {
  switch (p.dtype) {
    case DT_F32: launch_pipe_t<float>(p, grid, s, 0); break;
    case DT_BF16: launch_pipe_t<__nv_bfloat16>(p, grid, s, 1); break;
    case DT_F16: launch_pipe_t<__half>(p, grid, s, 2); break;
    default: throw std::runtime_error("dear: unsupported gradient dtype");
  }
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess)
    throw std::runtime_error(std::string("dear: launch of rs_pipe_kernel failed: ") + cudaGetErrorString(err));
}

}  // namespace dear
