// communicator.h — native communication runtime of the DeAR engine.
//
// `Communicator` is the H100 counterpart of the reference's NCCL+MPI
// `Communicator` class (common/comm_core/src/communicator.h:52-96): it owns the
// communication streams/events and exposes the same family of operations
// (bcast, reduce, allReduce, allReduceRB, allReduceRSAG, reduceScatter,
// allGather, sendrecv, synchronize, syncStream, getNumOfFreeStreams, barrier),
// but every operation is one of OUR kernels running over peer-mapped memory.
//
// `BucketSet` is the per-plan fused engine: symmetric parameter / gradient
// buckets plus the two fused kernels (reduce-scatter+scale in backward,
// SGD+all-gather in forward) that implement the decoupled all-reduce of
// dear/dear_dopt.py:242-372 without NCCL and without per-parameter kernels.
#pragma once
#include <torch/extension.h>
#include <cuda_runtime_api.h>

#include <atomic>
#include <memory>
#include <optional>
#include <string>
#include <vector>

#include "dear_common.h"
#include "symm_mem.h"

namespace dear {

struct CommOptions {
  int provider = static_cast<int>(Provider::CUDA_IPC);
  bool multicast = false;
  int device = -1;                       // -1 => host emulation
  int64_t staging_bytes = 32ll << 20;    // per stream slot
  int nstreams = 1;
  double spin_timeout_s = 20.0;          // in-kernel bounded spin
  double rendezvous_timeout_s = 120.0;
  int rs_grid = 96;
  int ag_grid = 96;
  int gen_grid = 8;
  // Kernel A variant per bucket: -1 = pick by bucket size (one-shot below `pipe_min_bytes`, stripe-pipelined TMA
  // pull above, NVLS ld_reduce only on request); 0 / 1 / 2 force RS_ALGO_ONESHOT / _PIPE / _NVLS for every bucket.
  int rs_algo = -1;
  int64_t pipe_min_bytes = int64_t(1) << 60;   // auto never picks the pipelined variant unless this is lowered
  int rs_grid_big = 128;                       // CTA bound for buckets >= big_bucket_bytes (their pack phase scales
  int64_t big_bucket_bytes = 128ll << 20;      // with the CTA count)
  int64_t stripe_target_bytes = 8ll << 20;   // bucket bytes per stripe the pipelined kernel aims for
  bool separate_ag_stream = true;            // all-gathers on their own stream (reference: three communicators)
};

class Communicator : public std::enable_shared_from_this<Communicator> {
 public:
  Communicator(int rank, int world, c10::intrusive_ptr<c10d::Store> store, std::string name,
               CommOptions opt);
  ~Communicator();

  int rank() const { return rank_; }
  int size() const { return world_; }
  bool is_cuda() const { return opt_.device >= 0; }
  bool has_multicast() const { return !arenas_.empty() && arenas_[0]->has_multicast(); }
  // Grow to at least `n` stream slots (collective: every rank calls it with the same n).  Each slot owns a stream,
  // two events and its own symmetric staging arena, so operations on different slots never serialise — the
  // reference's _extendComms (common/comm_core/src/communicator.cpp:85-95) creates one NCCL communicator per slot.
  void extend_streams(int n);
  int num_streams() const { return static_cast<int>(slots_.size()); }
  const CommOptions& options() const { return opt_; }
  const c10::intrusive_ptr<c10d::Store>& store() const { return store_; }
  const std::string& name() const { return name_; }

  // ---- collective ops (return the stream-slot "handle" like the reference) ----
  int allreduce_(torch::Tensor t, double scale);
  int allreduce_rsag_(torch::Tensor t, double scale);
  int allreduce_rb_(torch::Tensor t, double scale);
  int bcast_(torch::Tensor t, int root);
  int reduce_(torch::Tensor t, int root, double scale);
  int reduce_scatter(torch::Tensor send, torch::Tensor recv, double scale);
  int allgather(torch::Tensor send, torch::Tensor recv);
  int sendrecv(torch::Tensor send, torch::Tensor recv, int peer);
  int device_barrier();

  // ---- stream sync API (reference communicator.cpp:97-128) ----
  void synchronize();                 // host blocks on every comm stream
  void sync_stream(int handle);       // host blocks on one comm stream
  void wait_stream(int handle);       // current stream waits (no host block)
  int num_free_streams();
  void barrier();                     // host-side barrier through the store

  // Throws if a kernel flagged a spin-wait timeout.
  void check_status();
  int64_t launches() const { return launches_.load(); }
  void count_launch(int n = 1) { launches_.fetch_add(n); }

  std::string unique_key(const std::string& what);
  uint64_t timeout_ns() const { return static_cast<uint64_t>(opt_.spin_timeout_s * 1e9); }
  ArenaOptions arena_options() const;

 private:
  struct Slot {
    void* stream = nullptr;   // cudaStream_t
    void* ev_in = nullptr;    // cudaEvent_t
    void* ev_out = nullptr;
  };
  void add_slot();
  int run_gen(int op, const void* src, void* dst, uint64_t nelems, int dtype, uint32_t elem_bytes,
              int root_or_peer, float scale);
  int next_slot();
  void gen_chunked(int slot, int op, const char* src, char* dst, uint64_t nelems, int dtype,
                   uint32_t elem_bytes, int root_or_peer, float scale, uint64_t dst_stride_elems);

  int rank_, world_;
  c10::intrusive_ptr<c10d::Store> store_;
  std::string name_;
  CommOptions opt_;
  std::vector<std::shared_ptr<SymmArena>> arenas_;   // per-slot staging for the general ops
  std::vector<Slot> slots_;
  int cur_slot_ = 0;
  int key_seq_ = 0;
  int barrier_seq_ = 0;
  std::atomic<int64_t> launches_{0};
};

class BucketSet {
 public:
  // `grad_dtype` (default: `dtype`) is the element type of the gradient buckets.  An fp32 set may send its gradients
  // as bf16 / fp16: the pack rounds them, the pull accumulates in fp32 (a "converting" set, world > 1 only).
  BucketSet(std::shared_ptr<Communicator> comm, std::vector<int64_t> padded_numels, int dtype,
            bool with_grad_buckets, std::optional<int> grad_dtype = std::nullopt);
  ~BucketSet();

  int num_buckets() const { return static_cast<int>(buckets_.size()); }
  torch::Tensor param_buffer(int g);
  torch::Tensor grad_buffer(int g);
  bool has_multicast() const { return arena_->has_multicast(); }
  bool converting() const { return gdtype_ != dtype_; }

  // optimizer state shards of bucket g: momentum (SGD / RMSprop buffer, Adam exp_avg), var (Adam exp_avg_sq, RMSprop
  // square_avg), grad_avg (centered RMSprop); absent ones as None
  void set_shards(int g, torch::Tensor grad_shard, std::optional<torch::Tensor> mom,
                  std::optional<torch::Tensor> master, std::optional<torch::Tensor> var,
                  std::optional<torch::Tensor> grad_avg = std::nullopt);
  // number of updates already applied to bucket g (Adam bias correction); device-resident afterwards
  void set_step(int g, int64_t t);
  // Gradient sources for the fused pack.  Returns true if the device table was re-uploaded.
  bool set_pack(int g, const std::vector<int64_t>& src_ptrs, const std::vector<int64_t>& dst_off_bytes,
                const std::vector<int64_t>& nbytes, const std::vector<int64_t>& flags);
  bool set_hyper(int g, const std::vector<int64_t>& ends, const std::vector<double>& lr,
                 const std::vector<double>& wd, const std::vector<double>& mom,
                 const std::vector<double>& damp, const std::vector<int64_t>& nesterov,
                 const std::vector<int64_t>& opt, const std::vector<double>& beta2, const std::vector<double>& eps);

  void reduce_scatter(int g, bool pack);
  // extra factor folded into the 1/P of Kernel A's epilogue (static loss scaling: 1/S un-scales the gradients)
  void set_grad_scale(double s) { grad_scale_ = static_cast<float>(s); }
  // (algorithm, stripes, grid) chosen for bucket g at construction time: {"algo": "oneshot|pipe|nvls", ...}
  std::string rs_plan(int g) const;
  // the pipelined kernel's work list of bucket g as rows (src, dst_off, nbytes, stripe, flags) — for tests / debugging
  std::vector<std::vector<int64_t>> pack_pieces(int g) const;
  // `decide`: the step's deciding update (a scaler's skip decision, the clipping coefficient); needs the entry rendezvous
  void allgather_update(int g, bool do_update, bool first_step, bool entry_barrier, bool zero_grad, bool decide = false);
  // Dynamic loss scaling: `state` is the engine's AmpState (int32[9], on this set's device), or None for the static path.
  void set_amp(std::optional<torch::Tensor> state);
  // Global-norm clipping: `state` is the engine's ClipState (float32, clip_state_floats(nslots) elements, on this set's
  // device) and `slots[g]` the engine-wide slot of local bucket g; None switches clipping off.
  void set_clip(std::optional<torch::Tensor> state, const std::vector<int64_t>& slots);
  // The next update kernel on this set's all-gather stream waits for everything queued so far on both streams of
  // `other` (one decision per step across the sets of an engine).
  void join(BucketSet& other);
  void fence_current_to_comm();
  void wait_bucket(int g);
  void wait_rs(int g);
  void wait_all();
  void synchronize();
  int64_t comm_stream_handle() const { return reinterpret_cast<int64_t>(stream_); }

 private:
  struct Bucket {
    int64_t padded = 0;
    int64_t shard = 0;
    size_t param_off = 0, grad_off = 0;
    torch::Tensor grad_shard, mom, master, var, gavg;
    bool adam = false;
    bool rmsprop = false;
    bool rms_momentum = false;            // some RMSprop segment has momentum > 0: needs the momentum shard
    bool rms_centered = false;            // some RMSprop segment is centered: needs the grad_avg shard
    std::vector<PackSeg> pack_host;
    std::vector<HyperSeg> hyper_host;
    uint32_t ntiles = 0;
    bool pack_inplace = false;
    PackSeg* pack_dev = nullptr;
    size_t pack_cap = 0;
    // stripe-pipelined Kernel A: stripe-major list of <= 32 KB copies derived from pack_host (set_pack)
    std::vector<PackSeg> pieces_host;
    uint32_t piece_first[17] = {0};
    HyperSeg* hyper_dev = nullptr;
    size_t hyper_cap = 0;
    // Host staging of the two device tables.  Each table kind has its OWN double-buffered pinned area, and an
    // upload requested during a CUDA-graph capture fills a device table of its own (BucketSet::upload).
    struct Staging {
      void* pinned[2] = {nullptr, nullptr};
      size_t cap[2] = {0, 0};
      void* ev[2] = {nullptr, nullptr};
      int next = 0;
    };
    Staging stage_pack, stage_hyper;
    std::vector<void*> captured_tables;   // device tables owned by CUDA-graph captures; freed with the BucketSet
    void* capture_table = nullptr;        // table of the capture in progress (launch parameter of its kernels)
    bool eager_table_stale = false;       // pack_host mirrors a capture's table: the next eager set_pack must upload
    int rs_algo = RS_ALGO_ONESHOT;
    uint32_t nstripes = 1;
    uint64_t stripe_bytes = 0;
    int rs_grid = 1;
    void* ev_in = nullptr;
    void* rs_done = nullptr;
    void* ag_done = nullptr;
    bool ag_pending = false, rs_pending = false;
    bool ag_done_captured = false;   // ag_done was last recorded inside a CUDA-graph capture
  };
  void upload(Bucket& b, bool is_pack, const void* host, size_t bytes, void** dev, size_t* cap);
  int grid_for(int64_t shard_elems, int max_grid) const;

  std::shared_ptr<Communicator> comm_;
  std::shared_ptr<SymmArena> arena_;
  std::vector<Bucket> buckets_;
  int dtype_;
  int gdtype_;                  // gradient-bucket dtype (== dtype_ unless the set converts fp32 gradients)
  bool with_grad_;
  void* stream_ = nullptr;      // cudaStream_t (high priority): reduce-scatters, table uploads
  void* ag_stream_ = nullptr;   // cudaStream_t: update + all-gather kernels (== stream_ unless separate_ag_stream)
  void* ev_fence_ = nullptr;
  void* ev_fence_ag_ = nullptr;
  void* upload_stream_ = nullptr;   // private non-capturing stream for tables built during a capture
  float grad_scale_ = 1.0f;
  torch::Tensor amp_;               // AmpState of the engine's dynamic loss scaler (undefined: static path)
  torch::Tensor clip_;              // ClipState of the engine's global-norm clipping (undefined: no clipping)
  std::vector<uint32_t> clip_slot_; // engine-wide slot of each local bucket
  void* ev_join_ = nullptr;
};

// device launchers (kernels.cu) and host emulation (emu.cpp)
void launch_rs(const RSParams& p, int grid, cudaStream_t s);
void launch_rs_pipe(const RSParams& p, int grid, cudaStream_t s);
void launch_ag(const AGParams& p, int grid, cudaStream_t s);
void launch_gen(const GenParams& p, int grid, cudaStream_t s);
void emu_rs(const RSParams& p);
void emu_ag(const AGParams& p);
void emu_gen(const GenParams& p);

int dtype_of(const torch::Tensor& t);

}  // namespace dear
