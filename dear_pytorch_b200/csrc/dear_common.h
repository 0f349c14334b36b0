// dear_common.h — shared declarations for the H100-native DeAR runtime.
//
// Everything in this header is usable from host C++ and from sm_90a device
// code: the host-emulation backend (emu.cpp, used for CPU/gloo plumbing
// tests) and the CUDA kernels (kernels.cu) share the SAME argument structs
// and the SAME per-element math, so a CPU test of the emulation backend
// validates the indexing/SGD logic that the kernels execute.
//
// Parity notes (reference = lzhangbv/dear_pytorch):
//   * reduce-scatter call site  : dear/tensorfusion.py:475-476 -> comm_core reduceScatter
//   * all-gather call site      : dear/tensorfusion.py:477-478 -> comm_core allGather
//   * per-parameter SGD update  : dear/dear_dopt.py:310-336
// Here both collectives are fused with their adjacent elementwise work and
// run over peer-mapped (NVLink / NVSwitch) memory instead of NCCL.
#pragma once
#include <cstdint>
#include <cstddef>
#include <cmath>

#if defined(__CUDACC__)
#define DEAR_HD __host__ __device__ __forceinline__
#else
#define DEAR_HD inline
#endif

namespace dear {

constexpr int kMaxRanks = 16;            // one NVSwitch domain (8 on HGX H100)
constexpr int kNumChannels = 4096;       // signal-pad channels per arena
constexpr int kChannelsPerBucket = 4;    // RS_READY, RS_DONE, AG_ARRIVE, AG_PUSHED
constexpr int kGeneralChannels = 64;     // channels [0,64) are for general ops
constexpr uint32_t kPackTileBytes = 65536;
constexpr size_t kSignalPadBytes = size_t(kNumChannels) * kMaxRanks * sizeof(uint32_t);

// Channel ids for the general-purpose ops (all-reduce, broadcast, ...).
enum GeneralChannel : uint32_t {
  CH_BARRIER = 0,
  CH_AR_READY = 2,
  CH_AR_DONE = 3,
  CH_BCAST_READY = 4,
  CH_BCAST_DONE = 5,
  CH_REDUCE_READY = 6,
  CH_REDUCE_DONE = 7,
  CH_SENDRECV_READY = 8,
  CH_SENDRECV_DONE = 9,
  CH_AG_READY = 10,
  CH_AG_DONE = 11,
};

enum BucketChannel : uint32_t { RS_READY = 0, RS_DONE = 1, AG_ARRIVE = 2, AG_PUSHED = 3 };

DEAR_HD uint32_t bucket_channel(uint32_t bucket, uint32_t which) {
  return kGeneralChannels + bucket * kChannelsPerBucket + which;
}

// Error codes written to the (host-mapped) status word when a spin-wait
// times out.  A kernel never hangs the GPU: it gives up, flags, and exits.
enum Status : uint32_t {
  ST_OK = 0,
  ST_TIMEOUT_RS_READY = 1,
  ST_TIMEOUT_RS_DONE = 2,
  ST_TIMEOUT_AG_ARRIVE = 3,
  ST_TIMEOUT_AG_PUSHED = 4,
  ST_TIMEOUT_GENERAL = 5,
};

enum DType : int { DT_F32 = 0, DT_BF16 = 1, DT_F16 = 2 };

DEAR_HD size_t dtype_size(int dt) { return dt == DT_F32 ? 4 : 2; }

struct PeerTable {
  void* ptr[kMaxRanks];
};

// One gradient segment of a bucket (== one parameter's gradient).
// In a converting set (fp32 parameters whose gradients travel as bf16 / fp16, RSParams::src_f32) `dst_off` and
// `nbytes` count bucket (wire) bytes, and the pack reads the fp32 source at twice those offsets and byte counts.
struct PackSeg {
  const void* src;        // local gradient storage; nullptr => nothing to copy
  uint64_t dst_off;       // byte offset inside the bucket
  uint64_t nbytes;        // bytes to copy
  uint32_t tile_begin;    // exclusive prefix sum of 64 KiB tiles
  uint32_t flags;         // bit0: zero-fill the destination (gradient absent)
};
constexpr uint32_t SEG_ZERO_FILL = 1u;

// Contiguous element range of a bucket sharing one set of optimizer hyper-parameters.
enum OptKind : uint32_t { OPT_SGD = 0, OPT_ADAM = 1 /* L2 in the gradient */, OPT_ADAMW = 2 /* decoupled decay */ };
struct HyperSeg {
  uint64_t end;           // exclusive end (element offset within the bucket)
  float lr;
  float weight_decay;
  float momentum;         // SGD momentum, or Adam beta1
  float dampening;
  uint32_t nesterov;      // bit0: Nesterov momentum; bit1 (HYPER_SKIP): this rank saw no gradient for the range in
                          // this step — where the REDUCED gradient is exactly zero too (absent on every rank), leave
                          // parameter and state untouched, like torch.optim skips ``p.grad is None``
  uint32_t opt;           // OptKind
  float beta2;            // Adam only
  float eps;              // Adam only
};

constexpr uint32_t HYPER_NESTEROV = 1u;
constexpr uint32_t HYPER_SKIP = 2u;

// ---- per-element math shared by the CUDA kernels and the host emulation ----

// torch-1.8 SGD semantics (reference dear/dear_dopt.py:310-336):
//   g <- g + wd*p ; buf <- (first ? g : m*buf + (1-damp)*g) ; g <- nesterov ? g + m*buf : buf
//   p <- p - lr*g
// `g` is already averaged (the 1/P scale is fused into the reduce-scatter).  `coef` is the global-norm clipping
// coefficient (1 without clipping); it is applied after the HYPER_SKIP test, so a parameter without a gradient on any
// rank stays untouched even when `coef` is not finite.
DEAR_HD float sgd_update(float p, float g, float& mom, const HyperSeg& h, bool first_step,
                         bool has_mom_buf, float coef) {
  if ((h.nesterov & HYPER_SKIP) && g == 0.f) return p;
  g = g * coef;
  if (h.weight_decay != 0.f) g = g + h.weight_decay * p;
  if (h.momentum > 0.f && has_mom_buf) {
    float buf = first_step ? g : (h.momentum * mom + (1.f - h.dampening) * g);
    mom = buf;
    g = (h.nesterov & HYPER_NESTEROV) ? (g + h.momentum * buf) : buf;
  }
  return p - h.lr * g;
}

// torch.optim.Adam / AdamW semantics (non-amsgrad): exp_avg `m`, exp_avg_sq `v`, bias corrections
// bc1 = 1 - beta1^t, bc2 = 1 - beta2^t.  This extends the reference, whose DeAR path is SGD-only
// (dear/dear_dopt.py:310-336; its BERT driver had to drop AdamW, dear/bert_benchmark.py:118-122).
DEAR_HD float adam_update(float p, float g, float& m, float& v, const HyperSeg& h, float bc1, float sqrt_bc2,
                          float coef) {
  if ((h.nesterov & HYPER_SKIP) && g == 0.f) return p;
  g = g * coef;                                    // clipping coefficient, as in sgd_update
  if (h.opt == OPT_ADAM && h.weight_decay != 0.f) g = g + h.weight_decay * p;
  m = h.momentum * m + (1.f - h.momentum) * g;
  v = h.beta2 * v + (1.f - h.beta2) * g * g;
#if defined(__CUDA_ARCH__)
  const float denom = sqrtf(v) / sqrt_bc2 + h.eps;
#else
  const float denom = std::sqrt(v) / sqrt_bc2 + h.eps;
#endif
  if (h.opt == OPT_ADAMW) p = p * (1.f - h.lr * h.weight_decay);
  return p - (h.lr / bc1) * (m / denom);
}

// Index of the hyper segment containing element `e` (segments sorted by end).
DEAR_HD uint32_t find_hyper(const HyperSeg* segs, uint32_t n, uint64_t e) {
  uint32_t lo = 0, hi = n - 1;
  while (lo < hi) {
    uint32_t mid = (lo + hi) >> 1;
    if (e < segs[mid].end) hi = mid; else lo = mid + 1;
  }
  return lo;
}

// Index of the pack segment owning tile `t` (tile_begin is a prefix sum).
DEAR_HD uint32_t find_pack_seg(const PackSeg* segs, uint32_t n, uint32_t t) {
  uint32_t lo = 0, hi = n;          // invariant: segs[lo].tile_begin <= t
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (segs[mid].tile_begin <= t) lo = mid; else hi = mid;
  }
  return lo;
}

// ---- dynamic loss scaling -----------------------------------------------------

// Device-resident state of a dynamic loss scaler (parallel/grad_scaler.py), one per engine, shared by every BucketSet.
// Kernel A divides the reduced gradient by `scale` and ORs a non-finite result into `overflow`; the deciding Kernel B of
// the step agrees on the bit with every rank at its entry rendezvous, writes `found_inf`, applies torch's
// growth / backoff rule to `scale` and `growth_tracker`, and clears `overflow`.  Nine 32-bit words (torch int32[9]).
struct AmpState {
  uint32_t overflow;        // this rank saw a non-finite reduced gradient in the current step
  uint32_t found_inf;       // decision of the current step (some rank overflowed: skip the update)
  float scale;
  int32_t growth_tracker;
  uint32_t applied;         // updates applied so far (skipped steps excluded)
  float growth_factor;
  float backoff_factor;
  int32_t growth_interval;
  int32_t prev_growth_tracker;  // growth_tracker before the current step's rule (update(new_scale) restores it)
};

// torch._amp_update_scale_: back off on overflow, grow after `growth_interval` clean steps in a row.
DEAR_HD void amp_update_scale(AmpState* a, bool found_inf) {
  a->prev_growth_tracker = a->growth_tracker;
  if (found_inf) {
    a->scale *= a->backoff_factor;
    a->growth_tracker = 0;
    return;
  }
  const int32_t successful = a->growth_tracker + 1;
  if (successful == a->growth_interval) {
    const float grown = a->scale * a->growth_factor;
    if (grown - grown == 0.f) a->scale = grown;     // finite
    a->growth_tracker = 0;
  } else {
    a->growth_tracker = successful;
  }
}

// ---- global gradient-norm clipping ----------------------------------------------
//
// Device-resident state of `norm_clip` (torch.nn.utils.clip_grad_norm_ semantics), one per engine, shared by every
// BucketSet.  Buckets are numbered engine-wide ("slots").  Kernel A adds the square of every fp32 value it writes into
// a per-thread sum, reduces it over the CTA, stores the CTA's partial, and the last CTA of the bucket sums the
// partials in CTA order into the bucket's slot.  The step's deciding Kernel B sums the slots in slot order (this rank's
// partial), exchanges partials at its entry rendezvous, and every CTA of every rank sums them in rank order, so all
// ranks form the same `total_norm` and `coef` bit for bit.  The header is followed by float slot[nslots] and
// float cta[nslots][kClipMaxCtas].
constexpr uint32_t kClipMaxCtas = 1024;   // per-CTA partials per slot: Kernel A's grid may not exceed this with clipping
struct ClipState {
  float max_norm;
  float total_norm;         // 2-norm of the step's averaged (unscaled) gradient, before clipping
  float coef;               // min(1, max_norm / (total_norm + 1e-6)); NaN stays NaN, as in torch
  uint32_t nslots;
};

DEAR_HD float* clip_slots(ClipState* c) { return reinterpret_cast<float*>(c + 1); }
DEAR_HD float* clip_cta_partials(ClipState* c, uint32_t slot) {
  return clip_slots(c) + c->nslots + size_t(slot) * kClipMaxCtas;
}
DEAR_HD size_t clip_state_floats(uint32_t nslots) { return sizeof(ClipState) / 4 + size_t(nslots) * (1 + kClipMaxCtas); }

// torch: clip_coef = max_norm / (total_norm + 1e-6); clamp(max=1).  A comparison, not fminf: a NaN norm gives a NaN
// coefficient, like torch.clamp.
DEAR_HD float clip_coef(float max_norm, float total_norm) {
  const float c = max_norm / (total_norm + 1e-6f);
  return c > 1.f ? 1.f : c;
}

// The deciding kernel's partial sum of squares travels to every peer in a general channel of the bucket arena,
// written before the AG_ARRIVE release store and read after its acquire.  Two channels by epoch parity: a rank can
// write step s+1's partial while a peer still reads step s's (it cannot get to step s+2 before every peer arrived at
// step s+1, which follows that peer's step-s decision on its all-gather stream).
constexpr uint32_t CH_CLIP_PARTIAL = 12;   // and 13
DEAR_HD uint32_t clip_channel(uint32_t epoch) { return CH_CLIP_PARTIAL + (epoch & 1u); }

// ---- kernel parameter blocks ------------------------------------------------

// Kernel A: fused [pack local grads -> symmetric bucket] + cross-GPU ready
// barrier + pull-reduce of this rank's shard from every peer + 1/P scale.
struct RSParams {
  PeerTable grad;          // every rank's bucket base (grad[rank] is local)
  void* mc_grad;           // NVLS multicast alias of the bucket (or nullptr)
  float* out;              // local fp32 reduced shard [shard_elems]
  uint64_t shard_elems;    // elements per shard (bucket = world * shard_elems)
  float scale;             // 1/world
  const PackSeg* segs;     // device table (nullptr => nothing to pack)
  uint32_t nseg;
  uint32_t ntiles;
  PeerTable sig;           // every rank's signal pad (sig[rank] is local)
  uint32_t* ctrl;          // local control block: epoch[kNumChannels], counter[kNumChannels]
  uint32_t bucket;         // bucket id (selects channels)
  uint32_t direct_out;     // world==1 && fp32: pack straight into `out`, skip the pull phase
  int rank;
  int world;
  int dtype;               // DType of the gradient bucket
  uint32_t* status;        // host-mapped status word
  uint64_t timeout_ns;
  // stripe-pipelined variant (rs_pipe.cu): the shard is cut into `nstripes` stripes of `stripe_bytes`
  // (a multiple of kPipePackPiece); stripe k of EVERY shard is packed and published before stripe k+1
  uint32_t nstripes;
  uint32_t clip_slot;      // engine-wide bucket number: Kernel A's sum of squares goes to clip_slots(clip)[clip_slot]
  uint64_t stripe_bytes;
  // pack work list of the pipelined variant: `pieces` (device) holds <= kPipePackPiece-byte copies in stripe-major
  // order, stripe k owning entries [piece_first[k], piece_first[k+1])
  const PackSeg* pieces;
  uint32_t piece_first[17];
  // dynamic loss scale (nullptr => static path): the output is additionally divided by amp->scale, and a non-finite
  // output value sets amp->overflow
  AmpState* amp;
  // global-norm clipping (nullptr => no clipping): sum of squares of the written shard into the bucket's slot
  ClipState* clip;
  // converting set: the gradients are fp32 and the pack rounds them to `dtype` (round to nearest even) on the way
  // into the bucket; the pull is the ordinary 16-bit one.  Never set at world 1 (one rank has no wire).
  uint32_t src_f32;
};

// RS_READY flag encoding shared by both reduce-scatter kernels: (epoch << 8) | stripes_published; the one-shot
// kernel publishes kAllStripes.  Monotonic, so the wrap-safe ">=" wait works for either producer.
constexpr uint32_t kAllStripes = 255u;
constexpr uint32_t kMaxStripes = 16u;
constexpr uint32_t kPipeChunk = 16384;        // bytes per TMA bulk copy of the pull ring
constexpr uint32_t kPipePackPiece = 32768;    // bytes per pack work item

enum RsAlgo : int {
  RS_ALGO_ONESHOT = 0,    // pack, one cross-GPU flag round, pull with 128-bit loads (small buckets: fewest sync rounds)
  RS_ALGO_PIPE = 1,       // stripe-pipelined: pack warps + TMA (cp.async.bulk) pull ring + shared-memory reduce
  RS_ALGO_NVLS = 2,       // pack, then multimem.ld_reduce (the NVSwitch reduces); needs a multicast-bound arena
};

// Kernel B: fused [sharded SGD/momentum update] + push of the updated
// parameter shard into every peer's parameter bucket + completion barrier.
struct AGParams {
  PeerTable param;         // every rank's parameter bucket base
  void* mc_param;          // NVLS multicast alias (or nullptr)
  const float* grad_shard; // local fp32 averaged gradient shard
  float* mom_shard;        // local fp32 momentum / Adam exp_avg shard (nullptr if unused)
  float* var_shard;        // local fp32 Adam exp_avg_sq shard (nullptr for SGD)
  uint32_t* step_ctr;      // device-resident count of applied updates (Adam bias correction; graph-safe)
  uint32_t adam;           // 1 => every hyper segment is Adam/AdamW
  float* master_shard;     // local fp32 master shard (nullptr => param bucket is fp32 master)
  void* zero_grad;         // local gradient bucket to zero after use (nullptr => skip)
  uint64_t zero_bytes;
  uint64_t shard_elems;
  const HyperSeg* hyper;   // device table
  uint32_t nhyper;
  uint32_t first_step;     // momentum buffers are uninitialised (ignored with `amp`: then step_ctr == 0 decides)
  uint32_t entry_barrier;  // wait for every peer to reach this kernel before pushing
  uint32_t do_update;      // 0 => pure all-gather of the shard (no SGD)
  PeerTable sig;
  uint32_t* ctrl;
  uint32_t bucket;
  int rank;
  int world;
  int dtype;               // DType of the parameter bucket
  uint32_t* status;
  uint64_t timeout_ns;
  // dynamic loss scale (nullptr => static path): the update is skipped when amp->found_inf is set.  The deciding kernel
  // (`decide`, the engine's first update of the step, which has `entry_barrier`) carries amp->overflow in its
  // AG_ARRIVE flag, ORs every rank's bit and writes the decision.
  AmpState* amp;
  uint32_t decide;
  // global-norm clipping (nullptr => none): the deciding kernel forms clip->total_norm and clip->coef from every rank's
  // partial sum of squares; every update kernel of the step multiplies clip->coef into the gradient
  ClipState* clip;
};

// AG_ARRIVE flag encoding: (epoch << 1) | overflow bit of the sender (0 unless it is the deciding kernel).
DEAR_HD uint32_t arrive_flag(uint32_t epoch, uint32_t overflow) { return (epoch << 1) | (overflow ? 1u : 0u); }

// General ops on a symmetric staging buffer.
enum GenOp : int {
  GEN_ALLREDUCE = 0,   // sum over ranks of staging[0:n] -> dst (every rank)
  GEN_BCAST = 1,       // root's staging -> dst on every rank
  GEN_REDUCE = 2,      // sum over ranks -> dst on root only
  GEN_SENDRECV = 3,    // dst <- peer's staging
  GEN_ALLGATHER = 4,   // dst[r*n:(r+1)*n] <- rank r's staging
  GEN_BARRIER = 5,
  GEN_REDUCE_SCATTER = 6,  // dst[0:n/P] <- sum over ranks of staging[rank*n/P : ...]
};

struct GenParams {
  PeerTable stage;       // every rank's staging buffer
  void* mc_stage;
  const void* src;       // local input (copied into local staging first); may be nullptr
  void* dst;             // local output
  uint64_t nelems;       // elements of the op (per-rank input size)
  int op;
  int root_or_peer;
  float scale;           // applied to reductions
  uint32_t ready_chan;
  uint32_t done_chan;
  PeerTable sig;
  uint32_t* ctrl;
  int rank;
  int world;
  int dtype;             // DT_F32 / DT_BF16 / DT_F16 ; int64 is moved as raw bytes (no reduce)
  uint32_t elem_bytes;   // for raw moves
  uint64_t dst_stride_bytes;  // GEN_ALLGATHER: byte distance between ranks' slots in dst (0 => contiguous)
  uint32_t* status;
  uint64_t timeout_ns;
};

}  // namespace dear
