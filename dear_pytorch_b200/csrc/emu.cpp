// emu.cpp — host emulation of the three device kernels.
//
// Same parameter blocks, same flag protocol, same per-element math
// (dear_common.h), executed synchronously by the calling thread on POSIX
// shared memory.  It exists so that the complete runtime — rendezvous, arena
// layout, epochs, bucket state machine, sharded optimizer state — can be
// tested on a CPU-only box with several processes (tests/, gloo), and it is
// the executable specification the CUDA kernels are tested against.
#include <c10/util/BFloat16.h>
#include <c10/util/Half.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <thread>

#include "dear_common.h"

namespace dear {

namespace {

inline void flag_store_release(uint32_t* f, uint32_t v) { __atomic_store_n(f, v, __ATOMIC_RELEASE); }
inline uint32_t flag_load_acquire(const uint32_t* f) { return __atomic_load_n(f, __ATOMIC_ACQUIRE); }

inline uint32_t* flag_at(void* sig_base, uint32_t chan, int src) {
  return reinterpret_cast<uint32_t*>(sig_base) + size_t(chan) * kMaxRanks + src;
}

bool wait_flag(const uint32_t* f, uint32_t epoch, uint64_t timeout_ns, uint32_t* status, uint32_t code) {
  auto t0 = std::chrono::steady_clock::now();
  uint32_t spins = 0;
  while (static_cast<int32_t>(flag_load_acquire(f) - epoch) < 0) {
    if (++spins > 200) std::this_thread::sleep_for(std::chrono::microseconds(50));
    if ((spins & 0xff) == 0) {
      auto dt = std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now() - t0).count();
      if (static_cast<uint64_t>(dt) > timeout_ns) {
        if (status) __atomic_store_n(status, code, __ATOMIC_RELEASE);
        return false;
      }
    }
  }
  return true;
}

void wait_all(void* sig_local, uint32_t chan, uint32_t e, int world, uint64_t to, uint32_t* st, uint32_t code) {
  for (int r = 0; r < world; ++r) wait_flag(flag_at(sig_local, chan, r), e, to, st, code);
}
void signal_all(const PeerTable& sig, uint32_t chan, int rank, int world, uint32_t e) {
  for (int r = 0; r < world; ++r) flag_store_release(flag_at(sig.ptr[r], chan, rank), e);
}

template <typename T> inline float ld(const void* base, uint64_t i) {
  return static_cast<float>(reinterpret_cast<const T*>(base)[i]);
}
template <typename T> inline void st(void* base, uint64_t i, float v) {
  reinterpret_cast<T*>(base)[i] = static_cast<T>(v);
}

template <typename T>
void rs_impl(const RSParams& p) {
  void* sig_local = p.sig.ptr[p.rank];
  const uint32_t ch_ready = bucket_channel(p.bucket, RS_READY);
  const uint32_t ch_done = bucket_channel(p.bucket, RS_DONE);
  uint32_t* epoch_p = p.ctrl + ch_ready;
  const uint32_t e = *epoch_p + 1;
  const uint32_t e8 = e << 8;                    // RS_READY = (epoch << 8) | stripes published, like the device kernels
  wait_all(sig_local, ch_done, e - 1, p.world, p.timeout_ns, p.status, ST_TIMEOUT_RS_DONE);
  const uint64_t off = uint64_t(p.rank) * p.shard_elems;
  // 1/P (and 1/S of a static loss scale), times 1/scale of a dynamic one; a non-finite output sets amp->overflow
  const float scale = p.amp ? p.scale * (1.f / p.amp->scale) : p.scale;
  bool bad = false;
  float ss = 0.f;                                // clipping: sum of squares of the written shard, in element order
  auto put = [&](uint64_t i, float v) {
    p.out[i] = v;
    if (p.amp && !std::isfinite(v)) bad = true;
    if (p.clip) ss += v * v;
  };
  if (p.nstripes >= 1 && p.stripe_bytes > 0 && (p.pieces != nullptr || p.nstripes > 1)) {
    // stripe-pipelined variant (rs_pipe.cu): stripe k of every shard is packed from the stripe-major work list and
    // published; stripe k of my shard is reduced once every peer has published it
    char* bucket = reinterpret_cast<char*>(p.grad.ptr[p.rank]);
    for (uint32_t k = 0; k < p.nstripes; ++k) {
      if (p.pieces != nullptr) {
        for (uint32_t i = p.piece_first[k]; i < p.piece_first[k + 1]; ++i) {
          const PackSeg& pc = p.pieces[i];
          if (pc.flags & SEG_ZERO_FILL) std::memset(bucket + pc.dst_off, 0, pc.nbytes);
          else if (pc.src != nullptr) std::memcpy(bucket + pc.dst_off, pc.src, pc.nbytes);
        }
      }
      signal_all(p.sig, ch_ready, p.rank, p.world, e8 | (k + 1));
    }
    const uint64_t stripe_elems = p.stripe_bytes / sizeof(T);
    for (uint32_t k = 0; k < p.nstripes; ++k) {
      wait_all(sig_local, ch_ready, e8 | (k + 1), p.world, p.timeout_ns, p.status, ST_TIMEOUT_RS_READY);
      const uint64_t lo = uint64_t(k) * stripe_elems;
      const uint64_t hi = std::min<uint64_t>(p.shard_elems, lo + stripe_elems);
      for (uint64_t i = lo; i < hi; ++i) {
        // the kernel's order: peers rank+1, ..., P-1, 0, ..., rank-1 first, my own bucket last (rs_pipe.cu producer)
        float acc = 0.f;
        for (int j = 0; j < p.world; ++j) acc += ld<T>(p.grad.ptr[(p.rank + 1 + j) % p.world], off + i);
        put(i, acc * scale);
      }
    }
    if (bad) __atomic_fetch_or(&p.amp->overflow, 1u, __ATOMIC_RELAXED);
    if (p.clip) clip_slots(p.clip)[p.clip_slot] = ss;
    signal_all(p.sig, ch_done, p.rank, p.world, e);
    *epoch_p = e;
    return;
  }
  const bool direct = p.world == 1 && sizeof(T) == 4 && p.direct_out;
  // pack (tile by tile, exactly like the device kernel)
  if (p.segs != nullptr) {
    char* bucket = direct ? reinterpret_cast<char*>(p.out) : reinterpret_cast<char*>(p.grad.ptr[p.rank]);
    for (uint32_t tile = 0; tile < p.ntiles; ++tile) {
      const uint32_t si = find_pack_seg(p.segs, p.nseg, tile);
      const PackSeg& sg = p.segs[si];
      const uint64_t off2 = uint64_t(tile - sg.tile_begin) * kPackTileBytes;
      const uint64_t left = sg.nbytes - off2;
      const uint32_t nb = left < kPackTileBytes ? uint32_t(left) : kPackTileBytes;
      if (sg.flags & SEG_ZERO_FILL) {
        std::memset(bucket + sg.dst_off + off2, 0, nb);
      } else if (sg.src != nullptr && p.src_f32) {
        // converting set: fp32 source at twice the bucket offsets, rounded to T (c10's round to nearest even, as
        // torch's .to(): NaN stays NaN, fp16 overflow becomes inf)
        const float* src = reinterpret_cast<const float*>(sg.src) + off2 / sizeof(T);
        T* dst = reinterpret_cast<T*>(bucket + sg.dst_off + off2);
        for (uint32_t k = 0; k < nb / sizeof(T); ++k) dst[k] = static_cast<T>(src[k]);
      } else if (sg.src != nullptr && direct) {
        // fp32, one rank: the pack writes the reduced shard, so it applies the factor the reduction would have
        const float* src = reinterpret_cast<const float*>(reinterpret_cast<const char*>(sg.src) + off2);
        const uint64_t o = (sg.dst_off + off2) / sizeof(float);
        for (uint32_t k = 0; k < nb / sizeof(float); ++k) put(o + k, src[k] * scale);
      } else if (sg.src != nullptr) {
        std::memcpy(bucket + sg.dst_off + off2, reinterpret_cast<const char*>(sg.src) + off2, nb);
      }
    }
  }
  signal_all(p.sig, ch_ready, p.rank, p.world, e8 | kAllStripes);
  wait_all(sig_local, ch_ready, e8 | kAllStripes, p.world, p.timeout_ns, p.status, ST_TIMEOUT_RS_READY);
  for (uint64_t i = 0; i < p.shard_elems && !direct; ++i) {
    float acc = 0.f;
    for (int q = 0; q < p.world; ++q) acc += ld<T>(p.grad.ptr[q], off + i);   // fixed order
    put(i, acc * scale);
  }
  if (bad) __atomic_fetch_or(&p.amp->overflow, 1u, __ATOMIC_RELAXED);
  if (p.clip) clip_slots(p.clip)[p.clip_slot] = ss;
  signal_all(p.sig, ch_done, p.rank, p.world, e);
  *epoch_p = e;
}

template <typename T>
void ag_impl(const AGParams& p) {
  void* sig_local = p.sig.ptr[p.rank];
  const uint32_t ch_arrive = bucket_channel(p.bucket, AG_ARRIVE);
  const uint32_t ch_pushed = bucket_channel(p.bucket, AG_PUSHED);
  uint32_t* epoch_p = p.ctrl + ch_arrive;
  const uint32_t e = *epoch_p + 1;
  uint32_t found_inf = 0;
  const bool clip = p.clip && p.do_update;
  float coef = 1.f;
  if (p.entry_barrier) {
    // the deciding kernel's flags carry every rank's overflow bit (arrive_flag); OR them in rank order
    const uint32_t ov = (p.decide && p.amp) ? p.amp->overflow : 0u;
    if (clip && p.decide) {
      // this rank's partial sum of squares (slot order) goes to every peer before the AG_ARRIVE release store
      float t = 0.f;
      for (uint32_t i = 0; i < p.clip->nslots; ++i) t += clip_slots(p.clip)[i];
      uint32_t bits;
      std::memcpy(&bits, &t, 4);
      for (int r = 0; r < p.world; ++r) __atomic_store_n(flag_at(p.sig.ptr[r], clip_channel(e), p.rank), bits, __ATOMIC_RELAXED);
    }
    signal_all(p.sig, ch_arrive, p.rank, p.world, arrive_flag(e, ov));
    wait_all(sig_local, ch_arrive, arrive_flag(e, 0), p.world, p.timeout_ns, p.status, ST_TIMEOUT_AG_ARRIVE);
    if (clip && p.decide) {
      float t = 0.f;
      for (int r = 0; r < p.world; ++r) {
        flag_load_acquire(flag_at(sig_local, ch_arrive, r));
        const uint32_t bits = __atomic_load_n(flag_at(sig_local, clip_channel(e), r), __ATOMIC_RELAXED);
        float f;
        std::memcpy(&f, &bits, 4);
        t += f;
      }
      p.clip->total_norm = std::sqrt(t);
      p.clip->coef = clip_coef(p.clip->max_norm, p.clip->total_norm);
    }
    if (p.decide && p.amp) {
      for (int r = 0; r < p.world; ++r) found_inf |= flag_load_acquire(flag_at(sig_local, ch_arrive, r)) & 1u;
      p.amp->found_inf = found_inf;
      amp_update_scale(p.amp, found_inf != 0);
      if (!found_inf) p.amp->applied += 1;
      p.amp->overflow = 0;
    }
  }
  if (p.amp && !p.decide) found_inf = p.amp->found_inf;
  if (clip) coef = p.clip->coef;
  const bool upd = p.do_update && !found_inf;      // a skipped step is a pure all-gather of the unchanged shard
  const bool first_step = (p.amp && p.step_ctr) ? *p.step_ctr == 0 : p.first_step != 0;
  const uint64_t off = uint64_t(p.rank) * p.shard_elems;
  const bool has_mom = p.mom_shard != nullptr;
  const bool adam = p.adam && upd;
  const uint32_t t_step = (adam && p.step_ctr) ? *p.step_ctr + 1 : 1;
  for (uint64_t i = 0; i < p.shard_elems; ++i) {
    float pv = p.master_shard ? p.master_shard[i] : ld<T>(p.param.ptr[p.rank], off + i);
    if (upd) {
      const HyperSeg& h = p.hyper[p.nhyper == 1 ? 0 : find_hyper(p.hyper, p.nhyper, off + i)];
      if (adam) {
        const float bc1 = 1.f - std::pow(h.momentum, float(t_step));
        const float sqrt_bc2 = std::sqrt(1.f - std::pow(h.beta2, float(t_step)));
        pv = adam_update(pv, p.grad_shard[i], p.mom_shard[i], p.var_shard[i], h, bc1, sqrt_bc2, coef);
      } else {
        float mv = (has_mom && !first_step) ? p.mom_shard[i] : 0.f;
        pv = sgd_update(pv, p.grad_shard[i], mv, h, first_step, has_mom, coef);
        if (has_mom && h.momentum > 0.f) p.mom_shard[i] = mv;
      }
      if (p.master_shard) p.master_shard[i] = pv;
    }
    for (int k = 0; k < p.world; ++k) st<T>(p.param.ptr[(p.rank + k) % p.world], off + i, pv);
  }
  if (p.zero_grad) std::memset(p.zero_grad, 0, p.zero_bytes);
  signal_all(p.sig, ch_pushed, p.rank, p.world, e);
  wait_all(sig_local, ch_pushed, e, p.world, p.timeout_ns, p.status, ST_TIMEOUT_AG_PUSHED);
  *epoch_p = e;
  if (upd && p.step_ctr) *p.step_ctr = *p.step_ctr + 1;
}

template <typename T>
void reduce_from_peers(const GenParams& p, void* dst, uint64_t src_off, uint64_t n) {
  for (uint64_t i = 0; i < n; ++i) {
    float acc = 0.f;
    for (int q = 0; q < p.world; ++q) acc += ld<T>(p.stage.ptr[q], src_off + i);
    st<T>(dst, i, acc * p.scale);
  }
}

template <typename T>
void gen_impl(const GenParams& p) {
  void* sig_local = p.sig.ptr[p.rank];
  uint32_t* epoch_p = p.ctrl + p.ready_chan;
  const uint32_t e = *epoch_p + 1;
  const uint64_t nbytes = p.nelems * p.elem_bytes;
  wait_all(sig_local, p.done_chan, e - 1, p.world, p.timeout_ns, p.status, ST_TIMEOUT_GENERAL);
  const bool contributes = (p.op == GEN_ALLREDUCE) || (p.op == GEN_REDUCE) || (p.op == GEN_ALLGATHER) ||
                           (p.op == GEN_REDUCE_SCATTER) || (p.op == GEN_SENDRECV) ||
                           (p.op == GEN_BCAST && p.rank == p.root_or_peer);
  if (contributes && p.src && nbytes) std::memcpy(p.stage.ptr[p.rank], p.src, nbytes);
  signal_all(p.sig, p.ready_chan, p.rank, p.world, e);
  if (p.op == GEN_BCAST || p.op == GEN_SENDRECV)
    wait_flag(flag_at(sig_local, p.ready_chan, p.root_or_peer), e, p.timeout_ns, p.status, ST_TIMEOUT_GENERAL);
  else
    wait_all(sig_local, p.ready_chan, e, p.world, p.timeout_ns, p.status, ST_TIMEOUT_GENERAL);
  if (p.dst && nbytes) {
    switch (p.op) {
      case GEN_ALLREDUCE: reduce_from_peers<T>(p, p.dst, 0, p.nelems); break;
      case GEN_REDUCE: if (p.rank == p.root_or_peer) reduce_from_peers<T>(p, p.dst, 0, p.nelems); break;
      case GEN_REDUCE_SCATTER: {
        const uint64_t per = p.nelems / p.world;
        reduce_from_peers<T>(p, p.dst, per * p.rank, per);
        break;
      }
      case GEN_BCAST:
      case GEN_SENDRECV: std::memcpy(p.dst, p.stage.ptr[p.root_or_peer], nbytes); break;
      case GEN_ALLGATHER:
        for (int q = 0; q < p.world; ++q)
          std::memcpy(reinterpret_cast<char*>(p.dst) + uint64_t(q) * (p.dst_stride_bytes ? p.dst_stride_bytes : nbytes),
                      p.stage.ptr[q], nbytes);
        break;
      default: break;
    }
  }
  signal_all(p.sig, p.done_chan, p.rank, p.world, e);
  *epoch_p = e;
}

}  // namespace

void emu_rs(const RSParams& p) {
  switch (p.dtype) {
    case DT_BF16: rs_impl<c10::BFloat16>(p); break;
    case DT_F16: rs_impl<c10::Half>(p); break;
    default: rs_impl<float>(p); break;
  }
}
void emu_ag(const AGParams& p) {
  switch (p.dtype) {
    case DT_BF16: ag_impl<c10::BFloat16>(p); break;
    case DT_F16: ag_impl<c10::Half>(p); break;
    default: ag_impl<float>(p); break;
  }
}
void emu_gen(const GenParams& p) {
  switch (p.dtype) {
    case DT_BF16: gen_impl<c10::BFloat16>(p); break;
    case DT_F16: gen_impl<c10::Half>(p); break;
    default: gen_impl<float>(p); break;
  }
}

}  // namespace dear
