// bindings.cpp — pybind11 module `dear_pytorch_b200._C`.
//
// Counterpart of the reference's `comm_core` module
// (common/comm_core/src/comm_core.cpp:12-37): same operation family, but
// process bootstrap comes from torch.distributed's store (no MPI) and the data
// path is our own sm_90a kernels (no NCCL).
#include <torch/extension.h>
#include <torch/csrc/distributed/c10d/Store.hpp>

#include "communicator.h"

namespace py = pybind11;
using namespace dear;

namespace dear { namespace bn {
bool bn_act_supported(const torch::Tensor& x, const c10::optional<torch::Tensor>& residual);
int64_t bn_act_launches();
std::vector<torch::Tensor> bn_act_forward(const torch::Tensor& x, const c10::optional<torch::Tensor>& z,
                                          const c10::optional<torch::Tensor>& gamma, const c10::optional<torch::Tensor>& beta,
                                          c10::optional<torch::Tensor> running_mean, c10::optional<torch::Tensor> running_var,
                                          bool training, double momentum, double eps, bool relu);
std::vector<torch::Tensor> bn_act_backward(const torch::Tensor& dy, const torch::Tensor& x, const c10::optional<torch::Tensor>& y,
                                           const torch::Tensor& save_mean, const torch::Tensor& save_invstd,
                                           const torch::Tensor& scale, const torch::Tensor& shift, bool relu, bool has_residual);
} }

namespace dear { namespace ln {
bool ln_supported(const torch::Tensor& x, const c10::optional<torch::Tensor>& residual,
                  const c10::optional<torch::Tensor>& gamma, const c10::optional<torch::Tensor>& beta,
                  const c10::optional<torch::Tensor>& a_bias);
int64_t ln_launches();
std::vector<torch::Tensor> ln_forward(const torch::Tensor& a, const torch::Tensor& residual, const torch::Tensor& gamma,
                                      const torch::Tensor& beta, double p, bool training, double eps,
                                      const c10::optional<torch::Tensor>& a_bias);
std::vector<torch::Tensor> ln_backward(const torch::Tensor& dy, const torch::Tensor& s, const torch::Tensor& mean,
                                       const torch::Tensor& rstd, const torch::Tensor& gamma, const torch::Tensor& mask, double p,
                                       bool want_dbias);
bool bias_gelu_supported(const torch::Tensor& z, const c10::optional<torch::Tensor>& bias);
torch::Tensor bias_gelu_forward(const torch::Tensor& z, const torch::Tensor& bias);
std::vector<torch::Tensor> bias_gelu_backward(const torch::Tensor& dh, const torch::Tensor& z, const torch::Tensor& bias);
} }

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "H100-native DeAR communication runtime (fused reduce-scatter / SGD+all-gather kernels)";

  m.attr("MAX_RANKS") = kMaxRanks;
  m.attr("PROVIDER_HOST_SHM") = static_cast<int>(Provider::HOST_SHM);
  m.attr("PROVIDER_CUDA_IPC") = static_cast<int>(Provider::CUDA_IPC);
  m.attr("PROVIDER_CUDA_VMM") = static_cast<int>(Provider::CUDA_VMM);
  m.attr("SEG_ZERO_FILL") = static_cast<int>(SEG_ZERO_FILL);
  m.def("cuda_usable", &cuda_runtime_usable);
  m.def("status_word", [] { return static_cast<int64_t>(*status_word_host()); });
  m.def("_set_status_word", [](int64_t v) { *status_word_host() = static_cast<uint32_t>(v); },
        "fault injection for tests: pretend a kernel flagged a spin-wait timeout");

  py::class_<CommOptions>(m, "CommOptions")
      .def(py::init<>())
      .def_readwrite("provider", &CommOptions::provider)
      .def_readwrite("multicast", &CommOptions::multicast)
      .def_readwrite("device", &CommOptions::device)
      .def_readwrite("staging_bytes", &CommOptions::staging_bytes)
      .def_readwrite("nstreams", &CommOptions::nstreams)
      .def_readwrite("spin_timeout_s", &CommOptions::spin_timeout_s)
      .def_readwrite("rendezvous_timeout_s", &CommOptions::rendezvous_timeout_s)
      .def_readwrite("rs_grid", &CommOptions::rs_grid)
      .def_readwrite("ag_grid", &CommOptions::ag_grid)
      .def_readwrite("gen_grid", &CommOptions::gen_grid)
      .def_readwrite("rs_algo", &CommOptions::rs_algo)
      .def_readwrite("pipe_min_bytes", &CommOptions::pipe_min_bytes)
      .def_readwrite("rs_grid_big", &CommOptions::rs_grid_big)
      .def_readwrite("big_bucket_bytes", &CommOptions::big_bucket_bytes)
      .def_readwrite("stripe_target_bytes", &CommOptions::stripe_target_bytes)
      .def_readwrite("separate_ag_stream", &CommOptions::separate_ag_stream);

  py::class_<Communicator, std::shared_ptr<Communicator>>(m, "Communicator")
      .def(py::init([](int rank, int world, py::object store, std::string name, CommOptions opt) {
             c10::intrusive_ptr<c10d::Store> s;
             if (!store.is_none()) s = store.cast<c10::intrusive_ptr<c10d::Store>>();
             return std::make_shared<Communicator>(rank, world, s, std::move(name), opt);
           }),
           py::arg("rank"), py::arg("world"), py::arg("store"), py::arg("name"), py::arg("options"))
      .def("rank", &Communicator::rank)
      .def("size", &Communicator::size)
      .def("is_cuda", &Communicator::is_cuda)
      .def("has_multicast", &Communicator::has_multicast)
      .def("allReduce", &Communicator::allreduce_, py::arg("tensor"), py::arg("scale") = 1.0)
      .def("allReduceRSAG", &Communicator::allreduce_rsag_, py::arg("tensor"), py::arg("scale") = 1.0)
      .def("allReduceRB", &Communicator::allreduce_rb_, py::arg("tensor"), py::arg("scale") = 1.0)
      .def("bcast", &Communicator::bcast_, py::arg("tensor"), py::arg("root"))
      .def("reduce", &Communicator::reduce_, py::arg("tensor"), py::arg("root"), py::arg("scale") = 1.0)
      .def("extendStreams", &Communicator::extend_streams, py::arg("nstreams"))
      .def("numStreams", &Communicator::num_streams)
      .def("reduceScatter", &Communicator::reduce_scatter, py::arg("send"), py::arg("recv"), py::arg("scale") = 1.0)
      .def("allGather", &Communicator::allgather, py::arg("send"), py::arg("recv"))
      .def("sendrecv", &Communicator::sendrecv, py::arg("send"), py::arg("recv"), py::arg("peer"))
      .def("deviceBarrier", &Communicator::device_barrier)
      .def("synchronize", &Communicator::synchronize, py::call_guard<py::gil_scoped_release>())
      .def("syncStream", &Communicator::sync_stream, py::call_guard<py::gil_scoped_release>())
      .def("waitStream", &Communicator::wait_stream)
      .def("getNumOfFreeStreams", &Communicator::num_free_streams)
      .def("barrier", &Communicator::barrier, py::call_guard<py::gil_scoped_release>())
      .def("check_status", &Communicator::check_status)
      .def("launches", &Communicator::launches);

  py::class_<BucketSet, std::shared_ptr<BucketSet>>(m, "BucketSet")
      .def(py::init<std::shared_ptr<Communicator>, std::vector<int64_t>, int, bool, std::optional<int>>(), py::arg("comm"),
           py::arg("padded_numels"), py::arg("dtype"), py::arg("with_grad_buckets") = true,
           py::arg("grad_dtype") = py::none())
      .def("num_buckets", &BucketSet::num_buckets)
      .def("has_multicast", &BucketSet::has_multicast)
      .def("param_buffer", &BucketSet::param_buffer)
      .def("grad_buffer", &BucketSet::grad_buffer)
      .def("set_shards", &BucketSet::set_shards, py::arg("bucket"), py::arg("grad_shard"),
           py::arg("momentum") = py::none(), py::arg("master") = py::none(), py::arg("var") = py::none())
      .def("set_step", &BucketSet::set_step)
      .def("set_pack", &BucketSet::set_pack)
      .def("set_hyper", &BucketSet::set_hyper, py::arg("bucket"), py::arg("ends"), py::arg("lr"), py::arg("weight_decay"),
           py::arg("momentum"), py::arg("dampening"), py::arg("nesterov"), py::arg("opt") = std::vector<int64_t>{},
           py::arg("beta2") = std::vector<double>{}, py::arg("eps") = std::vector<double>{})
      .def("reduce_scatter", &BucketSet::reduce_scatter, py::arg("bucket"), py::arg("pack") = true)
      .def("rs_plan", &BucketSet::rs_plan, py::arg("bucket"))
      .def("set_grad_scale", &BucketSet::set_grad_scale, py::arg("scale"))
      .def("pack_pieces", &BucketSet::pack_pieces, py::arg("bucket"))
      .def("allgather_update", &BucketSet::allgather_update, py::arg("bucket"), py::arg("do_update") = true,
           py::arg("first_step") = false, py::arg("entry_barrier") = true, py::arg("zero_grad") = false,
           py::arg("decide") = false)
      .def("set_amp", &BucketSet::set_amp, py::arg("state"))
      .def("set_clip", &BucketSet::set_clip, py::arg("state"), py::arg("slots"))
      .def("join", &BucketSet::join, py::arg("other"))
      .def("fence_current_to_comm", &BucketSet::fence_current_to_comm)
      .def("wait_bucket", &BucketSet::wait_bucket)
      .def("wait_rs", &BucketSet::wait_rs)
      .def("wait_all", &BucketSet::wait_all)
      .def("synchronize", &BucketSet::synchronize, py::call_guard<py::gil_scoped_release>())
      .def("comm_stream_handle", &BucketSet::comm_stream_handle);

  // fused channels-last BatchNorm (+ residual) (+ ReLU)
  m.def("bn_act_supported", &dear::bn::bn_act_supported, py::arg("x"), py::arg("residual") = py::none());
  m.def("bn_act_launches", &dear::bn::bn_act_launches);
  m.def("bn_act_forward", &dear::bn::bn_act_forward, py::arg("x"), py::arg("residual"), py::arg("weight"), py::arg("bias"),
        py::arg("running_mean"), py::arg("running_var"), py::arg("training"), py::arg("momentum"), py::arg("eps"),
        py::arg("relu"));
  m.def("bn_act_backward", &dear::bn::bn_act_backward);

  // fused dropout + residual add + LayerNorm
  m.def("ln_supported", &dear::ln::ln_supported, py::arg("x"), py::arg("residual") = py::none(), py::arg("weight") = py::none(),
        py::arg("bias") = py::none(), py::arg("a_bias") = py::none());
  m.def("ln_launches", &dear::ln::ln_launches);
  m.def("ln_forward", &dear::ln::ln_forward, py::arg("a"), py::arg("residual"), py::arg("weight"), py::arg("bias"),
        py::arg("p"), py::arg("training"), py::arg("eps"), py::arg("a_bias") = py::none());
  m.def("ln_backward", &dear::ln::ln_backward, py::arg("dy"), py::arg("s"), py::arg("mean"), py::arg("rstd"), py::arg("weight"),
        py::arg("mask"), py::arg("p"), py::arg("want_dbias") = false);
  // fused bias + GELU (forward) and GELU backward + bias gradient (backward)
  m.def("bias_gelu_supported", &dear::ln::bias_gelu_supported, py::arg("z"), py::arg("bias") = py::none());
  m.def("bias_gelu_forward", &dear::ln::bias_gelu_forward);
  m.def("bias_gelu_backward", &dear::ln::bias_gelu_backward);

  // float32 elements of a ClipState for `nslots` buckets (BucketSet.set_clip); word 0 max_norm, 1 total_norm, 2 coef
  m.def("clip_state_floats", [](int64_t nslots) { return static_cast<int64_t>(clip_state_floats(static_cast<uint32_t>(nslots))); });
  m.attr("OPT_SGD") = static_cast<int>(OPT_SGD);
  m.attr("OPT_ADAM") = static_cast<int>(OPT_ADAM);
  m.attr("OPT_ADAMW") = static_cast<int>(OPT_ADAMW);
  m.attr("DT_F32") = static_cast<int>(DT_F32);
  m.attr("DT_BF16") = static_cast<int>(DT_BF16);
  m.attr("DT_F16") = static_cast<int>(DT_F16);
}
