// Python bindings of the tensor-core extension (dear_pytorch_b200._tc): the hand-written wgmma / TMA kernels of
// tc_ffn_hw.cu.
#include <torch/extension.h>

#include <atomic>

namespace py = pybind11;

namespace dear_tc {

static std::atomic<long> g_launches{0};

void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
long launches() { return g_launches.load(); }

std::vector<at::Tensor> ffn_up_hw(const at::Tensor& x, const at::Tensor& w, const at::Tensor& bias);   // tc_ffn_hw.cu
at::Tensor ffn_dgelu_hw(const at::Tensor& dy, const at::Tensor& wt, const at::Tensor& z);
at::Tensor ffn_dgelu_hw_nt(const at::Tensor& dy, const at::Tensor& w, const at::Tensor& z);
void set_ffn_hw_cluster(int cl);

}  // namespace dear_tc

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "hand-written sm_90a tensor-core kernels (wgmma / TMA) for the transformer feed-forward block";
  m.def("ffn_up_hw", &dear_tc::ffn_up_hw, py::arg("x"), py::arg("w"), py::arg("bias"),
        "H, Z = gelu(X W^T + b), X W^T + b   (X [M,K], W [N,K], b [N]; bf16, fp32 accumulate)");
  m.def("ffn_dgelu_hw", &dear_tc::ffn_dgelu_hw, py::arg("dy"), py::arg("wt"), py::arg("z"),
        "dZ = (dY Wt^T) * gelu'(Z), Wt = transposed down-projection weight [N, K] (K-major B operand)");
  m.def("ffn_dgelu_hw_nt", &dear_tc::ffn_dgelu_hw_nt, py::arg("dy"), py::arg("w"), py::arg("z"),
        "dZ = (dY W) * gelu'(Z) with W [K, N] as nn.Linear stores it (MN-major B operand, no transposed copy)");
  m.def("set_ffn_hw_cluster", &dear_tc::set_ffn_hw_cluster, py::arg("cl"),
        "CTAs per cluster sharing the B tile through TMA multicast: -1 = default (1); 1 / 2 / 4 forced (must divide the tile rows)");
  m.def("launches", &dear_tc::launches);
}
