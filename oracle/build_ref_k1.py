"""TEST INFRASTRUCTURE: builds the reference's own Hopper block-sparse forward (fastvideo-kernel/csrc/attention/
block_sparse_h100.cu, ThunderKittens wgmma, sm_90a) from the reference tree in $FVB_REFERENCE_ROOT into
oracle/_ref/k1_ref*.so (git-ignored) -- the kernel tests/test_gpu_vsa_golden.py compares ours against head to head.
Run where the reference sources lie:  FVB_REFERENCE_ROOT=<reference checkout> python -m oracle.build_ref_k1"""
import os

import torch.utils.cpp_extension as ce

REF = os.environ.get("FVB_REFERENCE_ROOT", "")
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    csrc = os.path.join(REF, "fastvideo-kernel", "csrc")
    src = os.path.join(csrc, "attention", "block_sparse_h100.cu")
    if not REF or not os.path.exists(src):
        print("reference sources not present; nothing built")
        return
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    out = os.path.join(HERE, "_ref")
    os.makedirs(out, exist_ok=True)
    tk = [os.path.join(REF, "fastvideo-kernel", d) for d in ("ThunderKittens/include", "ThunderKittens/prototype", "include")]
    try:
        ce.load(name="k1_ref", sources=[os.path.join(HERE, "k1_binding.cpp"), src], build_directory=out, is_python_module=False,
                extra_cuda_cflags=["-gencode", "arch=compute_90a,code=sm_90a", "-DKITTENS_HOPPER", "-O3", "-std=c++20",
                                   "--expt-relaxed-constexpr", "--expt-extended-lambda", "--use_fast_math"],
                extra_include_paths=[os.path.join(csrc, "attention"), *tk],
                extra_ldflags=["-L/usr/local/cuda/lib64/stubs", "-lcuda"], verbose=True)
    except (OSError, ImportError) as e:  # loading needs libcuda.so.1, absent on a CPU-only machine; the .so is built
        print("built (not loadable here):", e)
    print("built:", [f for f in os.listdir(out) if f.endswith(".so")])


if __name__ == "__main__":
    main()
