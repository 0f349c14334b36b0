// kernels.cu — sm_90a device code of the DeAR runtime.
//
// Kernel A (rs_kernel):   gradient pack + reduce-scatter + fp32 accumulate + 1/P scale
//                         replaces: bucket copy_ (dear/dear_dopt.py:265), ncclReduceScatter
//                         (common/comm_core/src/communicator.cpp:157-169) and div_ (:306).
// Kernel B (ag_kernel):   sharded SGD/momentum update + all-gather (push) of the updated
//                         parameter shard, replaces ncclAllGather (communicator.cpp:171-183),
//                         the copy-out / div_ / _sgd / fill_ per-parameter loop
//                         (dear/dear_dopt.py:293-336).
// gen_kernel:             small one-shot all-reduce / broadcast / reduce / sendrecv /
//                         all-gather / barrier on a symmetric staging buffer
//                         (communicator.cpp:130-155,185-242,287-304).
//
// Cross-GPU protocol: every rank owns a "signal pad" (uint32 flags indexed
// [channel][source rank]) inside its symmetric arena.  A producer publishes
// data with  stores -> bar.sync -> fence.sys -> st.release.sys(flag@peer, epoch)
// and a consumer observes it with ld.acquire.sys(flag@local) >= epoch followed
// by plain loads.  Epochs live in device memory (ctrl block) and are advanced
// by the last CTA of each kernel, so launches carry no host-side sequence
// number and are CUDA-graph replayable.  Spin waits are bounded: on timeout a
// status word in host-mapped memory is set and the kernel exits.
//
// Data moves over NVLink with 128-bit peer loads (pull, Kernel A) and 128-bit
// peer stores (push, Kernel B); when an NVLS multicast alias of the bucket is
// available the same kernels switch to multimem.ld_reduce / multimem.st so the
// NVSwitch performs the reduction / replication.
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdexcept>
#include <string>
#include "dear_common.h"
#include "dear_device.cuh"

namespace dear {

// ----------------------------------------------------------------------------
// Kernel A — pack + reduce-scatter + scale
// ----------------------------------------------------------------------------
constexpr int kPackVecPerThread = kPackTileBytes / 16 / kThreads;   // 8 x 128-bit per thread per tile

// AMP: dynamic loss scaling (p.amp != nullptr) — divide by the device-resident scale and test every written value for
// finiteness.  A separate instantiation, so the static path compiles to exactly the work it did without a scaler.
// CLIP: global-norm clipping (p.clip != nullptr) — add the square of every written value to a per-thread sum, which
// the exit folds into the bucket's slot (clip_store_cta_partial / clip_combine_slot).  Also a separate instantiation.
// CVT: a converting set (p.src_f32) — the gradients are fp32 and the pack rounds them to the 16-bit T of the bucket;
// the pull phase is the ordinary one of T.  Instantiated for W != 1 only.
template <typename T, int W, bool MC, bool AMP, bool CLIP, bool CVT = false>
__global__ void __launch_bounds__(kThreads, 1) rs_kernel(const RSParams p) {
  using Tr = ElemTraits<T>;
  constexpr int EV = Tr::kPerVec;
  __shared__ PackSeg s_segs[kMaxSmemSegs];

  const int tid = threadIdx.x;
  const int world = (W > 0) ? W : p.world;
  void* sig_local = p.sig.ptr[p.rank];
  const uint32_t ch_ready = bucket_channel(p.bucket, RS_READY);
  const uint32_t ch_done = bucket_channel(p.bucket, RS_DONE);
  uint32_t* epoch_p = p.ctrl + ch_ready;
  uint32_t* cnt_pack = p.ctrl + kNumChannels + ch_ready;
  uint32_t* cnt_exit = p.ctrl + kNumChannels + ch_done;
  const uint32_t e = *reinterpret_cast<volatile uint32_t*>(epoch_p) + 1;
  // single-GPU fast path: the "reduction" of one rank is a copy (fp32) or a widening conversion (bf16 / fp16),
  // so the pack writes the fp32 shard (== the whole bucket) directly and the pull phase disappears.
  const bool direct = (W == 1) && p.direct_out;
  const bool direct16 = direct && sizeof(T) == 2;
  // 1/P (and 1/S of a static loss scale), times 1/scale of a dynamic one
  const float scale = AMP ? p.scale * (1.f / *reinterpret_cast<volatile float*>(&p.amp->scale)) : p.scale;
  bool bad = false;                               // AMP: this thread wrote a non-finite value
  float ss = 0.f;                                 // CLIP: sum of squares of the values this thread wrote

  // (0) my bucket may still be read by a peer's previous reduce-scatter.
  wait_all_peers(sig_local, ch_done, e - 1, world, p.timeout_ns, p.status, ST_TIMEOUT_RS_DONE);

  // (1) pack: copy this rank's gradients into the symmetric bucket (64 KiB tiles, 8 independent
  //     128-bit loads in flight per thread).
  if (p.segs != nullptr && p.ntiles > 0) {
    const bool in_smem = p.nseg <= kMaxSmemSegs;
    if (in_smem) {
      for (uint32_t i = tid; i < p.nseg; i += kThreads) s_segs[i] = p.segs[i];
      __syncthreads();
    }
    const PackSeg* segs = in_smem ? s_segs : p.segs;
    char* bucket = direct ? reinterpret_cast<char*>(p.out) : reinterpret_cast<char*>(p.grad.ptr[p.rank]);
    for (uint32_t tile = blockIdx.x; tile < p.ntiles; tile += gridDim.x) {
      const uint32_t si = find_pack_seg(segs, p.nseg, tile);
      const PackSeg sg = segs[si];
      const uint64_t off = uint64_t(tile - sg.tile_begin) * kPackTileBytes;
      const uint64_t left = sg.nbytes - off;
      const uint32_t nb = left < kPackTileBytes ? uint32_t(left) : kPackTileBytes;
      char* d = bucket + sg.dst_off + off;
      const uint32_t nvec = nb >> 4;
      if (direct16) {
        // 16-bit gradients, one GPU: widen straight into the fp32 shard (element e of the bucket = out[e])
        float* o = p.out + ((sg.dst_off + off) >> 1);
        const bool zero = (sg.flags & SEG_ZERO_FILL) != 0;
        if (!zero && sg.src == nullptr) continue;
        const char* s = reinterpret_cast<const char*>(sg.src) + off;
        uint4 r[kPackVecPerThread];
#pragma unroll
        for (int k = 0; k < kPackVecPerThread; ++k) {
          const uint32_t v = tid + k * kThreads;
          r[k] = make_uint4(0, 0, 0, 0);
          if (v < nvec && !zero) r[k] = ld_stream(s + (size_t(v) << 4));
        }
#pragma unroll
        for (int k = 0; k < kPackVecPerThread; ++k) {
          const uint32_t v = tid + k * kThreads;
          if (v < nvec) {
            float f[8];
            Tr::unpack(r[k], f);
#pragma unroll
            for (int x = 0; x < 8; ++x) f[x] *= scale;
            if (AMP) bad |= !all_finite<8>(f);
            if (CLIP) ss += sum_sq<8>(f);
            float4* o4 = reinterpret_cast<float4*>(o + size_t(v) * 8);
            o4[0] = make_float4(f[0], f[1], f[2], f[3]);
            o4[1] = make_float4(f[EV - 4], f[EV - 3], f[EV - 2], f[EV - 1]);
          }
        }
        for (uint32_t b = (nvec << 4) + tid * 2; b < nb; b += kThreads * 2) {
          const float x = zero ? 0.f : Tr::from_raw16(*reinterpret_cast<const uint16_t*>(s + b)) * scale;
          if (AMP) bad |= !isfinite(x);
          if (CLIP) ss += x * x;
          o[b >> 1] = x;
        }
        continue;
      }
      if (sg.flags & SEG_ZERO_FILL) {
        const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int k = 0; k < kPackVecPerThread; ++k) {
          const uint32_t v = tid + k * kThreads;
          if (v < nvec) st_stream(d + (size_t(v) << 4), z);
        }
        for (uint32_t b = (nvec << 4) + tid * 2; b < nb; b += kThreads * 2)
          *reinterpret_cast<uint16_t*>(d + b) = 0;
      } else if (CVT && sg.src != nullptr) {
        // fp32 source, 16-bit bucket: a tile is kPackTileBytes of the bucket and twice that of the source.  Two 128-bit
        // fp32 loads make one 128-bit store of 8 rounded elements (16 loads in flight per thread).
        const char* s = reinterpret_cast<const char*>(sg.src) + 2 * off;
        uint4 r[kPackVecPerThread][2];
#pragma unroll
        for (int k = 0; k < kPackVecPerThread; ++k) {
          const uint32_t v = tid + k * kThreads;
          if (v < nvec) {
            r[k][0] = ld_stream(s + (size_t(v) << 5));
            r[k][1] = ld_stream(s + (size_t(v) << 5) + 16);
          }
        }
#pragma unroll
        for (int k = 0; k < kPackVecPerThread; ++k) {
          const uint32_t v = tid + k * kThreads;
          if (v < nvec) {
            float f[8];
            ElemTraits<float>::unpack(r[k][0], f);
            ElemTraits<float>::unpack(r[k][1], f + 4);
            st_stream(d + (size_t(v) << 4), Tr::pack(f));
          }
        }
        for (uint32_t b = (nvec << 4) + tid * 2; b < nb; b += kThreads * 2)
          *reinterpret_cast<uint16_t*>(d + b) = Tr::to_raw16(*reinterpret_cast<const float*>(s + 2 * size_t(b)));
      } else if (sg.src != nullptr) {
        const char* s = reinterpret_cast<const char*>(sg.src) + off;
        uint4 r[kPackVecPerThread];
#pragma unroll
        for (int k = 0; k < kPackVecPerThread; ++k) {
          const uint32_t v = tid + k * kThreads;
          if (v < nvec) r[k] = ld_stream(s + (size_t(v) << 4));
        }
        if (direct) {
          // fp32 gradients, one GPU: the pack writes the fp32 shard, so it applies the factor the pull phase would have
#pragma unroll
          for (int k = 0; k < kPackVecPerThread; ++k) {
            const uint32_t v = tid + k * kThreads;
            if (v < nvec) {
              float f[4] = {__uint_as_float(r[k].x) * scale, __uint_as_float(r[k].y) * scale,
                            __uint_as_float(r[k].z) * scale, __uint_as_float(r[k].w) * scale};
              if (AMP) bad |= !all_finite<4>(f);
              if (CLIP) ss += sum_sq<4>(f);
              st_stream(d + (size_t(v) << 4),
                        make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3])));
            }
          }
          for (uint32_t b = (nvec << 4) + tid * 4; b < nb; b += kThreads * 4) {
            const float x = *reinterpret_cast<const float*>(s + b) * scale;
            if (AMP) bad |= !isfinite(x);
            if (CLIP) ss += x * x;
            *reinterpret_cast<float*>(d + b) = x;
          }
          continue;
        }
#pragma unroll
        for (int k = 0; k < kPackVecPerThread; ++k) {
          const uint32_t v = tid + k * kThreads;
          if (v < nvec) st_stream(d + (size_t(v) << 4), r[k]);
        }
        for (uint32_t b = (nvec << 4) + tid * 2; b < nb; b += kThreads * 2)
          *reinterpret_cast<uint16_t*>(d + b) = *reinterpret_cast<const uint16_t*>(s + b);
      }
    }
  }

  // (2) publish "bucket packed" to every peer once ALL my CTAs are done packing.
  if (grid_arrive_is_last(cnt_pack)) {
    signal_all_peers(p.sig, ch_ready, p.rank, world, (e << 8) | kAllStripes);
    if (tid == 0) *cnt_pack = 0;
  }

  // (3) wait until every peer's bucket is packed.
  wait_all_peers(sig_local, ch_ready, (e << 8) | kAllStripes, world, p.timeout_ns, p.status, ST_TIMEOUT_RS_READY);

  // (4) pull-reduce my shard from every peer; fp32 accumulate; fused 1/P scale.
  if (!direct) {
    const uint64_t nvec = p.shard_elems / EV;
    const uint64_t shard_byte_off = uint64_t(p.rank) * p.shard_elems * sizeof(T);
    const uint64_t gstride = uint64_t(gridDim.x) * kThreads;
    if (MC) {
      const char* mc = reinterpret_cast<const char*>(p.mc_grad) + shard_byte_off;
      constexpr int U = 8;
      for (uint64_t v0 = uint64_t(blockIdx.x) * kThreads + tid; v0 < nvec; v0 += gstride * U) {
        uint4 r[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint64_t v = v0 + u * gstride;
          if (v < nvec) r[u] = Tr::mc_reduce(mc + (v << 4));
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint64_t v = v0 + u * gstride;
          if (v < nvec) {
            float f[EV];
            Tr::unpack(r[u], f);
#pragma unroll
            for (int k = 0; k < EV; ++k) f[k] *= scale;
            if (AMP) bad |= !all_finite<EV>(f);
            if (CLIP) ss += sum_sq<EV>(f);
            float4* o = reinterpret_cast<float4*>(p.out + v * EV);
            o[0] = make_float4(f[0], f[1], f[2], f[3]);
            if (EV == 8) o[1] = make_float4(f[EV - 4], f[EV - 3], f[EV - 2], f[EV - 1]);
          }
        }
      }
    } else if (W > 0) {
      constexpr int WW = W > 0 ? W : 1;
      constexpr int U = (WW >= 8) ? 2 : (WW == 4 ? 4 : 8);     // U*W >= 16 loads in flight per thread
      for (uint64_t v0 = uint64_t(blockIdx.x) * kThreads + tid; v0 < nvec; v0 += gstride * U) {
        uint4 r[U][WW];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint64_t v = v0 + u * gstride;
#pragma unroll
          for (int q = 0; q < WW; ++q) {
            if (v < nvec) {
              const char* base = reinterpret_cast<const char*>(p.grad.ptr[q]) + shard_byte_off;
              r[u][q] = ld_peer(base + (v << 4));
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint64_t v = v0 + u * gstride;
          if (v < nvec) {
            float acc[EV];
#pragma unroll
            for (int k = 0; k < EV; ++k) acc[k] = 0.f;
#pragma unroll
            for (int q = 0; q < WW; ++q) {   // fixed order => run-to-run deterministic
              float f[EV];
              Tr::unpack(r[u][q], f);
#pragma unroll
              for (int k = 0; k < EV; ++k) acc[k] += f[k];
            }
#pragma unroll
            for (int k = 0; k < EV; ++k) acc[k] *= scale;
            if (AMP) bad |= !all_finite<EV>(acc);
            if (CLIP) ss += sum_sq<EV>(acc);
            float4* o = reinterpret_cast<float4*>(p.out + v * EV);
            o[0] = make_float4(acc[0], acc[1], acc[2], acc[3]);
            if (EV == 8) o[1] = make_float4(acc[EV - 4], acc[EV - 3], acc[EV - 2], acc[EV - 1]);
          }
        }
      }
    } else {
      constexpr int U = 2;
      for (uint64_t v0 = uint64_t(blockIdx.x) * kThreads + tid; v0 < nvec; v0 += gstride * U) {
        float acc[U][EV];
#pragma unroll
        for (int u = 0; u < U; ++u)
#pragma unroll
          for (int k = 0; k < EV; ++k) acc[u][k] = 0.f;
        for (int q = 0; q < world; ++q) {
          const char* base = reinterpret_cast<const char*>(p.grad.ptr[q]) + shard_byte_off;
#pragma unroll
          for (int u = 0; u < U; ++u) {
            const uint64_t v = v0 + u * gstride;
            if (v < nvec) {
              float f[EV];
              Tr::unpack(ld_peer(base + (v << 4)), f);
#pragma unroll
              for (int k = 0; k < EV; ++k) acc[u][k] += f[k];
            }
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const uint64_t v = v0 + u * gstride;
          if (v < nvec) {
#pragma unroll
            for (int k = 0; k < EV; ++k) acc[u][k] *= scale;
            if (AMP) bad |= !all_finite<EV>(acc[u]);
            if (CLIP) ss += sum_sq<EV>(acc[u]);
            float4* o = reinterpret_cast<float4*>(p.out + v * EV);
            o[0] = make_float4(acc[u][0], acc[u][1], acc[u][2], acc[u][3]);
            if (EV == 8) o[1] = make_float4(acc[u][EV - 4], acc[u][EV - 3], acc[u][EV - 2], acc[u][EV - 1]);
          }
        }
      }
    }
  }

  // AMP: one atomic per CTA into this rank's overflow word (read by the step's deciding Kernel B)
  if (AMP) {
    if (__syncthreads_or(bad) && tid == 0) atomicOr(&p.amp->overflow, 1u);
  }
  if (CLIP) clip_store_cta_partial(p.clip, p.clip_slot, ss);

  // (5) tell every peer I am done reading its bucket; advance the epoch.
  if (grid_arrive_is_last(cnt_exit)) {
    signal_all_peers(p.sig, ch_done, p.rank, world, e);
    if (tid == 0) {
      if (CLIP) clip_combine_slot(p.clip, p.clip_slot);
      *cnt_exit = 0;
      *epoch_p = e;
    }
  }
}

// ----------------------------------------------------------------------------
// Kernel B — sharded SGD + all-gather push
// ----------------------------------------------------------------------------
__device__ __forceinline__ void ld_f32x(const float* base, uint64_t v, int ev, float* out) {
  const float4* m = reinterpret_cast<const float4*>(base + v * ev);
  const float4 a = m[0];
  out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
  if (ev == 8) {
    const float4 b = m[1];
    out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
  }
}
__device__ __forceinline__ void st_f32x(float* base, uint64_t v, int ev, const float* in) {
  float4* m = reinterpret_cast<float4*>(base + v * ev);
  m[0] = make_float4(in[0], in[1], in[2], in[3]);
  if (ev == 8) m[1] = make_float4(in[4], in[5], in[6], in[7]);
}

// CLIP: global-norm clipping (p.clip != nullptr): multiply the step's coefficient into the gradient.  A separate
// instantiation, so the path without clipping compiles as before.
template <typename T, int W, bool MC, bool ADAM, bool CLIP>
__global__ void __launch_bounds__(kThreads, 1) ag_kernel(const AGParams p) {
  using Tr = ElemTraits<T>;
  constexpr int EV = Tr::kPerVec;
  constexpr int EVA = 8;                        // register array length (>= EV)
  constexpr int U = ADAM ? ((EV == 4) ? 2 : 1) : ((EV == 4) ? 4 : 2);   // vectors in flight per thread
  __shared__ HyperSeg s_hyper[kMaxSmemHyper];

  const int tid = threadIdx.x;
  const int world = (W > 0) ? W : p.world;
  void* sig_local = p.sig.ptr[p.rank];
  const uint32_t ch_arrive = bucket_channel(p.bucket, AG_ARRIVE);
  const uint32_t ch_pushed = bucket_channel(p.bucket, AG_PUSHED);
  uint32_t* epoch_p = p.ctrl + ch_arrive;
  uint32_t* cnt_exit = p.ctrl + kNumChannels + ch_pushed;
  const uint32_t e = *reinterpret_cast<volatile uint32_t*>(epoch_p) + 1;

  const bool hyper_smem = p.nhyper <= kMaxSmemHyper;
  if (p.do_update && hyper_smem) {
    for (uint32_t i = tid; i < p.nhyper; i += kThreads) s_hyper[i] = p.hyper[i];
  }
  const HyperSeg* hyper = hyper_smem ? s_hyper : p.hyper;

  // (0) nobody may overwrite a peer's parameters before that peer finished the
  // backward pass that still reads them: rendezvous at kernel entry.  With a dynamic loss scale the deciding kernel's
  // flags carry every rank's overflow bit: each CTA ORs them (fixed rank order), so all ranks reach the same decision.
  AmpState* const amp = p.amp;
  ClipState* const clip = p.clip;
  uint32_t found_inf = 0;
  float coef = 1.f;                               // CLIP: the step's clipping coefficient
  if (p.entry_barrier) {
    if (blockIdx.x == 0) {
      // (with CLIP the deciding kernel may run without a scaler)
      const bool amp_decide = p.decide && (!CLIP || amp != nullptr);
      const uint32_t ov = (amp_decide && tid < world) ? *reinterpret_cast<volatile uint32_t*>(&amp->overflow) : 0u;
      if (CLIP && p.decide) {
        // this rank's partial: its slots in slot order.  Thread q stores it into peer q's pad and then, in
        // signal_all_peers, fences and release-stores the AG_ARRIVE flag: a peer that acquires the flag sees the partial.
        __shared__ float s_partial;
        if (tid == 0) {
          const volatile float* slots = clip_slots(clip);
          float t = 0.f;
          for (uint32_t i = 0; i < clip->nslots; ++i) t += slots[i];
          s_partial = t;
        }
        __syncthreads();
        if (tid < world)
          *reinterpret_cast<volatile uint32_t*>(flag_at(p.sig.ptr[tid], clip_channel(e), p.rank)) = __float_as_uint(s_partial);
      }
      signal_all_peers(p.sig, ch_arrive, p.rank, world, arrive_flag(e, ov));
    }
    wait_all_peers(sig_local, ch_arrive, arrive_flag(e, 0), world, p.timeout_ns, p.status, ST_TIMEOUT_AG_ARRIVE);
    if (p.decide && (!CLIP || amp != nullptr)) {
      const uint32_t bit = tid < world ? (ld_acquire_sys(flag_at(sig_local, ch_arrive, tid)) & 1u) : 0u;
      found_inf = __syncthreads_or(bit) ? 1u : 0u;
      if (blockIdx.x == 0 && tid == 0) {
        amp->found_inf = found_inf;
        amp_update_scale(amp, found_inf != 0);
        if (!found_inf) amp->applied += 1;
        amp->overflow = 0;            // the next step's reduce-scatters are stream-ordered after this kernel
      }
    }
    if (CLIP && p.decide) {
      // every CTA of every rank sums the same W partials in rank order: one total and one coefficient everywhere
      __shared__ float s_coef;
      if (tid == 0) {
        float t = 0.f;
        for (int q = 0; q < world; ++q) {
          const uint32_t* f = flag_at(sig_local, clip_channel(e), q);
          (void)ld_acquire_sys(flag_at(sig_local, ch_arrive, q));
          t += __uint_as_float(*reinterpret_cast<const volatile uint32_t*>(f));
        }
        const float total = sqrtf(t);
        s_coef = clip_coef(clip->max_norm, total);
        if (blockIdx.x == 0) {
          clip->total_norm = total;
          clip->coef = s_coef;
        }
      }
      __syncthreads();
      coef = s_coef;
    }
  } else {
    __syncthreads();
  }
  // the step's other update kernels follow the deciding one on the all-gather stream(s)
  if (amp != nullptr && !p.decide) found_inf = *reinterpret_cast<volatile uint32_t*>(&amp->found_inf);
  if (CLIP && !p.decide) coef = *reinterpret_cast<volatile float*>(&clip->coef);
  // a skipped step is a pure all-gather of the unchanged shard: same flag rounds, gradient bucket still zeroed
  const bool upd = p.do_update && !found_inf;
  // with a dynamic loss scale the host cannot know which update is the first one applied: count on the device
  const bool first_step = (amp != nullptr && p.step_ctr != nullptr) ? *reinterpret_cast<volatile uint32_t*>(p.step_ctr) == 0
                                                                     : p.first_step != 0;

  // (1) update my shard and push it into every rank's parameter bucket.
  {
    const uint64_t nvec = p.shard_elems / EV;
    const uint64_t shard_elem_off = uint64_t(p.rank) * p.shard_elems;
    const uint64_t gstride = uint64_t(gridDim.x) * kThreads;
    const char* local_param = reinterpret_cast<const char*>(p.param.ptr[p.rank]);
    const bool has_mom = p.mom_shard != nullptr;
    const bool load_mom = has_mom && (ADAM || !first_step) && upd;
    // Adam bias corrections come from a device-resident update counter (graph replay safe)
    const uint32_t t_step = (ADAM && p.step_ctr != nullptr) ? *reinterpret_cast<volatile uint32_t*>(p.step_ctr) + 1 : 1;
    for (uint64_t v0 = uint64_t(blockIdx.x) * kThreads + tid; v0 < nvec; v0 += gstride * U) {
      float pv[U][EVA], gv[U][EVA], mv[U][EVA];
      float vv[ADAM ? U : 1][EVA];
      // ---- all loads first (memory-level parallelism) ----
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint64_t v = v0 + u * gstride;
        if (v < nvec) {
          if (p.master_shard != nullptr) {
            ld_f32x(p.master_shard, v, EV, pv[u]);
          } else {
            Tr::unpack(*reinterpret_cast<const uint4*>(local_param + (shard_elem_off + v * EV) * sizeof(T)), pv[u]);
          }
          if (upd) ld_f32x(p.grad_shard, v, EV, gv[u]);
          if (load_mom) {
            ld_f32x(p.mom_shard, v, EV, mv[u]);
          } else {
#pragma unroll
            for (int k = 0; k < EV; ++k) mv[u][k] = 0.f;
          }
          if (ADAM && upd) ld_f32x(p.var_shard, v, EV, vv[ADAM ? u : 0]);
        }
      }
      // ---- update + stores ----
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint64_t v = v0 + u * gstride;
        if (v < nvec) {
          const uint64_t ge = shard_elem_off + v * EV;     // element offset within the bucket
          if (upd) {
            const HyperSeg h = hyper[p.nhyper == 1 ? 0 : find_hyper(hyper, p.nhyper, ge)];
            if (ADAM) {
              const float bc1 = 1.f - powf(h.momentum, float(t_step));
              const float sqrt_bc2 = sqrtf(1.f - powf(h.beta2, float(t_step)));
#pragma unroll
              for (int k = 0; k < EV; ++k)
                pv[u][k] = adam_update(pv[u][k], gv[u][k], mv[u][k], vv[ADAM ? u : 0][k], h, bc1, sqrt_bc2,
                                       CLIP ? coef : 1.f);
              st_f32x(p.mom_shard, v, EV, mv[u]);
              st_f32x(p.var_shard, v, EV, vv[ADAM ? u : 0]);
            } else {
#pragma unroll
              for (int k = 0; k < EV; ++k)
                pv[u][k] = sgd_update(pv[u][k], gv[u][k], mv[u][k], h, first_step, has_mom, CLIP ? coef : 1.f);
              if (has_mom && h.momentum > 0.f) st_f32x(p.mom_shard, v, EV, mv[u]);
            }
            if (p.master_shard != nullptr) st_f32x(p.master_shard, v, EV, pv[u]);
          }
          const uint4 outv = Tr::pack(pv[u]);
          const uint64_t boff = ge * sizeof(T);
          if (MC) {
            multimem_st(reinterpret_cast<char*>(p.mc_param) + boff, outv);
          } else if (W > 0) {
#pragma unroll
            for (int k = 0; k < (W > 0 ? W : 1); ++k) {
              const int q = (p.rank + k) % (W > 0 ? W : 1);   // own copy first, then rotate over peers
              st_stream(reinterpret_cast<char*>(p.param.ptr[q]) + boff, outv);
            }
          } else {
            for (int k = 0; k < world; ++k) {
              const int q = (p.rank + k) % world;
              st_stream(reinterpret_cast<char*>(p.param.ptr[q]) + boff, outv);
            }
          }
        }
      }
    }
    // zero the consumed local gradient bucket (grad-as-bucket-view mode only).
    if (p.zero_grad != nullptr) {
      const uint64_t zvec = p.zero_bytes >> 4;
      const uint4 z = make_uint4(0, 0, 0, 0);
      char* zp = reinterpret_cast<char*>(p.zero_grad);
      for (uint64_t v = uint64_t(blockIdx.x) * kThreads + tid; v < zvec; v += gstride) st_stream(zp + (v << 4), z);
    }
  }

  // (2) once ALL my CTAs pushed: publish, then wait until every peer's shard has
  // landed here.  The kernel (and therefore the stream event the next forward
  // waits on) completes only when the whole bucket is up to date on this GPU.
  if (grid_arrive_is_last(cnt_exit)) {
    signal_all_peers(p.sig, ch_pushed, p.rank, world, e);
    wait_all_peers(sig_local, ch_pushed, e, world, p.timeout_ns, p.status, ST_TIMEOUT_AG_PUSHED);
    if (tid == 0) {
      *cnt_exit = 0;
      *epoch_p = e;
      if (upd && p.step_ctr != nullptr) *p.step_ctr = *p.step_ctr + 1;
    }
  }
}

// ----------------------------------------------------------------------------
// General ops on the symmetric staging buffer
// ----------------------------------------------------------------------------
__device__ __forceinline__ void copy_bytes_grid(void* dst, const void* src, uint64_t nbytes) {
  const uint64_t gtid = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t gstride = uint64_t(gridDim.x) * blockDim.x;
  const uintptr_t a = reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src);
  if ((a & 15) == 0) {
    const uint64_t nvec = nbytes >> 4;
    for (uint64_t v = gtid; v < nvec; v += gstride)
      st_stream(reinterpret_cast<char*>(dst) + (v << 4),
                ld_stream(reinterpret_cast<const char*>(src) + (v << 4)));
    for (uint64_t b = (nvec << 4) + gtid; b < nbytes; b += gstride)
      reinterpret_cast<char*>(dst)[b] = reinterpret_cast<const char*>(src)[b];
  } else if ((a & 3) == 0) {
    const uint64_t nw = nbytes >> 2;
    for (uint64_t v = gtid; v < nw; v += gstride)
      reinterpret_cast<uint32_t*>(dst)[v] = reinterpret_cast<const uint32_t*>(src)[v];
    for (uint64_t b = (nw << 2) + gtid; b < nbytes; b += gstride)
      reinterpret_cast<char*>(dst)[b] = reinterpret_cast<const char*>(src)[b];
  } else {
    for (uint64_t b = gtid; b < nbytes; b += gstride)
      reinterpret_cast<char*>(dst)[b] = reinterpret_cast<const char*>(src)[b];
  }
}

template <typename T> __device__ __forceinline__ float to_f32(T v);
template <> __device__ __forceinline__ float to_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f32<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }
template <> __device__ __forceinline__ float to_f32<__half>(__half v) { return __half2float(v); }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 from_f32<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half from_f32<__half>(float v) { return __float2half_rn(v); }

// dst[0:n] = scale * sum_q stage_q[src_off : src_off+n]   (fp32 accumulate, fixed order)
template <typename T>
__device__ __forceinline__ void reduce_from_peers(const GenParams& p, T* dst, uint64_t src_off,
                                                  uint64_t n) {
  using Tr = ElemTraits<T>;
  constexpr int EV = Tr::kPerVec;
  const uint64_t gtid = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const uint64_t gstride = uint64_t(gridDim.x) * blockDim.x;
  const bool aligned = ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) && ((src_off * sizeof(T)) & 15) == 0;
  uint64_t done = 0;
  if (aligned) {
    const uint64_t nvec = n / EV;
    for (uint64_t v = gtid; v < nvec; v += gstride) {
      float acc[EV];
#pragma unroll
      for (int k = 0; k < EV; ++k) acc[k] = 0.f;
      for (int q = 0; q < p.world; ++q) {
        float f[EV];
        Tr::unpack(ld_peer(reinterpret_cast<const char*>(p.stage.ptr[q]) + (src_off + v * EV) * sizeof(T)), f);
#pragma unroll
        for (int k = 0; k < EV; ++k) acc[k] += f[k];
      }
#pragma unroll
      for (int k = 0; k < EV; ++k) acc[k] *= p.scale;
      *reinterpret_cast<uint4*>(dst + v * EV) = Tr::pack(acc);
    }
    done = nvec * EV;
  }
  for (uint64_t i = done + gtid; i < n; i += gstride) {
    float acc = 0.f;
    for (int q = 0; q < p.world; ++q)
      acc += to_f32<T>(reinterpret_cast<const T*>(p.stage.ptr[q])[src_off + i]);
    dst[i] = from_f32<T>(acc * p.scale);
  }
}

template <typename T>
__global__ void __launch_bounds__(kThreads, 1) gen_kernel(const GenParams p) {
  const int tid = threadIdx.x;
  const int world = p.world;
  void* sig_local = p.sig.ptr[p.rank];
  uint32_t* epoch_p = p.ctrl + p.ready_chan;
  uint32_t* cnt_a = p.ctrl + kNumChannels + p.ready_chan;
  uint32_t* cnt_b = p.ctrl + kNumChannels + p.done_chan;
  const uint32_t e = *reinterpret_cast<volatile uint32_t*>(epoch_p) + 1;
  const uint64_t nbytes = p.nelems * p.elem_bytes;

  // (0) staging buffers are free once every peer finished the previous op.
  wait_all_peers(sig_local, p.done_chan, e - 1, world, p.timeout_ns, p.status, ST_TIMEOUT_GENERAL);

  // (1) stage my contribution.
  const bool contributes = (p.op == GEN_ALLREDUCE) || (p.op == GEN_REDUCE) || (p.op == GEN_ALLGATHER) ||
                           (p.op == GEN_REDUCE_SCATTER) || (p.op == GEN_SENDRECV) ||
                           (p.op == GEN_BCAST && p.rank == p.root_or_peer);
  if (contributes && p.src != nullptr && nbytes > 0) copy_bytes_grid(p.stage.ptr[p.rank], p.src, nbytes);

  // (2) publish.
  if (grid_arrive_is_last(cnt_a)) {
    signal_all_peers(p.sig, p.ready_chan, p.rank, world, e);
    if (tid == 0) *cnt_a = 0;
  }

  // (3) wait for the producers this op depends on.
  if (p.op == GEN_BCAST) {
    if (tid == 0) wait_flag(flag_at(sig_local, p.ready_chan, p.root_or_peer), e, p.timeout_ns, p.status, ST_TIMEOUT_GENERAL);
    __syncthreads();
  } else if (p.op == GEN_SENDRECV) {
    if (tid == 0) wait_flag(flag_at(sig_local, p.ready_chan, p.root_or_peer), e, p.timeout_ns, p.status, ST_TIMEOUT_GENERAL);
    __syncthreads();
  } else {
    wait_all_peers(sig_local, p.ready_chan, e, world, p.timeout_ns, p.status, ST_TIMEOUT_GENERAL);
  }

  // (4) the op itself.
  if (p.dst != nullptr && nbytes > 0) {
    switch (p.op) {
      case GEN_ALLREDUCE:
        reduce_from_peers<T>(p, reinterpret_cast<T*>(p.dst), 0, p.nelems);
        break;
      case GEN_REDUCE:
        if (p.rank == p.root_or_peer) reduce_from_peers<T>(p, reinterpret_cast<T*>(p.dst), 0, p.nelems);
        break;
      case GEN_REDUCE_SCATTER: {
        const uint64_t per = p.nelems / world;
        reduce_from_peers<T>(p, reinterpret_cast<T*>(p.dst), per * p.rank, per);
        break;
      }
      case GEN_BCAST:
      case GEN_SENDRECV:
        copy_bytes_grid(p.dst, p.stage.ptr[p.root_or_peer], nbytes);
        break;
      case GEN_ALLGATHER:
        for (int q = 0; q < world; ++q)
          copy_bytes_grid(reinterpret_cast<char*>(p.dst) + uint64_t(q) * (p.dst_stride_bytes ? p.dst_stride_bytes : nbytes),
                          p.stage.ptr[q], nbytes);
        break;
      default:
        break;
    }
  }

  // (5) done reading peers' staging; advance the epoch.
  if (grid_arrive_is_last(cnt_b)) {
    signal_all_peers(p.sig, p.done_chan, p.rank, world, e);
    if (tid == 0) {
      *cnt_b = 0;
      *epoch_p = e;
    }
  }
}

// Multi-tensor fused SGD for the single-GPU path is Kernel B with world == 1.

// ----------------------------------------------------------------------------
// launchers
// ----------------------------------------------------------------------------
static void check_launch(const char* what) {
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess)
    throw std::runtime_error(std::string("dear: launch of ") + what + " failed: " + cudaGetErrorString(err));
}

template <typename T, bool MC, bool AMP, bool CLIP, bool CVT>
static void launch_rs_wa(const RSParams& p, int grid, cudaStream_t s) {
  switch (p.world) {
    case 1:
      if constexpr (CVT) throw std::runtime_error("dear: a converting gradient set needs more than one rank");
      else rs_kernel<T, 1, MC, AMP, CLIP><<<grid, kThreads, 0, s>>>(p);
      break;
    case 2: rs_kernel<T, 2, MC, AMP, CLIP, CVT><<<grid, kThreads, 0, s>>>(p); break;
    case 4: rs_kernel<T, 4, MC, AMP, CLIP, CVT><<<grid, kThreads, 0, s>>>(p); break;
    case 8: rs_kernel<T, 8, MC, AMP, CLIP, CVT><<<grid, kThreads, 0, s>>>(p); break;
    default: rs_kernel<T, 0, MC, AMP, CLIP, CVT><<<grid, kThreads, 0, s>>>(p); break;
  }
}

template <typename T, bool MC, bool CVT = false>
static void launch_rs_w(const RSParams& p, int grid, cudaStream_t s) {
  const bool clip = p.clip != nullptr;
  if (p.amp != nullptr) clip ? launch_rs_wa<T, MC, true, true, CVT>(p, grid, s) : launch_rs_wa<T, MC, true, false, CVT>(p, grid, s);
  else clip ? launch_rs_wa<T, MC, false, true, CVT>(p, grid, s) : launch_rs_wa<T, MC, false, false, CVT>(p, grid, s);
}

void launch_rs(const RSParams& p, int grid, cudaStream_t s) {
  const bool mc = p.mc_grad != nullptr;
  if (p.src_f32) {
    switch (p.dtype) {
      case DT_BF16:
        mc ? launch_rs_w<__nv_bfloat16, true, true>(p, grid, s) : launch_rs_w<__nv_bfloat16, false, true>(p, grid, s);
        break;
      case DT_F16: mc ? launch_rs_w<__half, true, true>(p, grid, s) : launch_rs_w<__half, false, true>(p, grid, s); break;
      default: throw std::runtime_error("dear: a converting gradient set sends bf16 or fp16");
    }
    check_launch("rs_kernel");
    return;
  }
  switch (p.dtype) {
    case DT_F32: mc ? launch_rs_w<float, true>(p, grid, s) : launch_rs_w<float, false>(p, grid, s); break;
    case DT_BF16: mc ? launch_rs_w<__nv_bfloat16, true>(p, grid, s) : launch_rs_w<__nv_bfloat16, false>(p, grid, s); break;
    case DT_F16: mc ? launch_rs_w<__half, true>(p, grid, s) : launch_rs_w<__half, false>(p, grid, s); break;
    default: throw std::runtime_error("dear: unsupported gradient dtype");
  }
  check_launch("rs_kernel");
}

template <typename T, bool MC, bool ADAM, bool CLIP>
static void launch_ag_wa(const AGParams& p, int grid, cudaStream_t s) {
  switch (p.world) {
    case 1: ag_kernel<T, 1, MC, ADAM, CLIP><<<grid, kThreads, 0, s>>>(p); break;
    case 2: ag_kernel<T, 2, MC, ADAM, CLIP><<<grid, kThreads, 0, s>>>(p); break;
    case 4: ag_kernel<T, 4, MC, ADAM, CLIP><<<grid, kThreads, 0, s>>>(p); break;
    case 8: ag_kernel<T, 8, MC, ADAM, CLIP><<<grid, kThreads, 0, s>>>(p); break;
    default: ag_kernel<T, 0, MC, ADAM, CLIP><<<grid, kThreads, 0, s>>>(p); break;
  }
}

template <typename T, bool MC>
static void launch_ag_w(const AGParams& p, int grid, cudaStream_t s) {
  const bool adam = p.adam && p.do_update, clip = p.clip != nullptr && p.do_update;
  if (adam) clip ? launch_ag_wa<T, MC, true, true>(p, grid, s) : launch_ag_wa<T, MC, true, false>(p, grid, s);
  else clip ? launch_ag_wa<T, MC, false, true>(p, grid, s) : launch_ag_wa<T, MC, false, false>(p, grid, s);
}

void launch_ag(const AGParams& p, int grid, cudaStream_t s) {
  const bool mc = p.mc_param != nullptr;
  switch (p.dtype) {
    case DT_F32: mc ? launch_ag_w<float, true>(p, grid, s) : launch_ag_w<float, false>(p, grid, s); break;
    case DT_BF16: mc ? launch_ag_w<__nv_bfloat16, true>(p, grid, s) : launch_ag_w<__nv_bfloat16, false>(p, grid, s); break;
    case DT_F16: mc ? launch_ag_w<__half, true>(p, grid, s) : launch_ag_w<__half, false>(p, grid, s); break;
    default: throw std::runtime_error("dear: unsupported parameter dtype");
  }
  check_launch("ag_kernel");
}

void launch_gen(const GenParams& p, int grid, cudaStream_t s) {
  switch (p.dtype) {
    case DT_BF16: gen_kernel<__nv_bfloat16><<<grid, kThreads, 0, s>>>(p); break;
    case DT_F16: gen_kernel<__half><<<grid, kThreads, 0, s>>>(p); break;
    default: gen_kernel<float><<<grid, kThreads, 0, s>>>(p); break;
  }
  check_launch("gen_kernel");
}

}  // namespace dear
