// TEST INFRASTRUCTURE: minimal pybind module around the REFERENCE's Hopper block-sparse forward
// (fastvideo-kernel/csrc/attention/block_sparse_h100.cu, ThunderKittens, sm_90a), compiled in place from the reference tree
// by oracle/build_ref_k1.py into oracle/_ref/ (git-ignored). No reference source is copied.
#include <torch/extension.h>

#include <vector>

// q, k, v: [B, H, S_pad, 128] bf16; q2k_idx / q2k_num: the 64-block lists; returns {o, lse}
std::vector<torch::Tensor> block_sparse_fwd(torch::Tensor q, torch::Tensor k, torch::Tensor v, torch::Tensor q2k_block_sparse_index,
                                            torch::Tensor q2k_block_sparse_num, torch::Tensor variable_block_sizes);

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) { m.def("fwd", &block_sparse_fwd, "reference sm_90a VSA forward (64-token blocks, BHSD)"); }
