"""TEST INFRASTRUCTURE: makes the reference's own Triton kernel package available to the GPU box.

/root/reference does not exist on the GPU box and the reference's VSA kernels (fused_block_mean, fused_topk_mask,
map_to_index, the Triton block-sparse forward/backward) only run with a GPU driver, so they can serve as an oracle only
there. This script stages the *unmodified* Python package `fastvideo-kernel/python/fastvideo_kernel` from where it lies
under /root/reference into `oracle/_ref/fastvideo_kernel/` -- git-ignored (never enters the history), not
gpurun-ignored (travels to the box like oracle/_ref/k1_ref.so). `oracle/gen_golden_gpu.py` then imports it THERE to
write the fixtures `tests/golden/vsa_gpu_*.pt`.

Run in the build container:  python -m oracle.stage_ref_kernels
"""
import os
import shutil

REF = os.environ.get("FVB_REFERENCE_ROOT", "")
HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(REF, "fastvideo-kernel", "python", "fastvideo_kernel")
DST = os.path.join(HERE, "_ref", "fastvideo_kernel")
# the reference's own Python package (.py files only, without its tests / third_party trees), so that the CPU arm of
# bench.py can time the REFERENCE's WanTransformerBlock on the GPU box's host cores (cpu_baseline.kind = "reference")
SRC_FV = os.path.join(REF, "fastvideo")
DST_FV = os.path.join(HERE, "_ref", "reference_py", "fastvideo")


def main() -> bool:
    if not os.path.isdir(SRC):
        print("reference sources not present; nothing staged")
        return False
    if os.path.isdir(DST):
        shutil.rmtree(DST)
    shutil.copytree(SRC, DST, ignore=shutil.ignore_patterns("__pycache__", "*.pyc", "*.so"))
    n = sum(len(fs) for _, _, fs in os.walk(DST))
    print(f"staged {n} files of the reference's fastvideo_kernel package into {DST} (git-ignored)")
    if os.path.isdir(DST_FV):
        shutil.rmtree(DST_FV)

    def ignore(d, names):
        rel = os.path.relpath(d, SRC_FV)
        skip = {"__pycache__"}
        if rel == ".":
            skip |= {"tests"}
        if rel == "third_party":  # 261 MB of vendored eval / other-model code; platform detection needs pynvml.py only
            return [n_ for n_ in names if n_ not in ("__init__.py", "pynvml.py")]
        return [n_ for n_ in names if n_ in skip or (os.path.isfile(os.path.join(d, n_)) and not n_.endswith(".py"))]

    shutil.copytree(SRC_FV, DST_FV, ignore=ignore)
    n = sum(len(fs) for _, _, fs in os.walk(DST_FV))
    print(f"staged {n} .py files of the reference's fastvideo package into {DST_FV} (git-ignored)")
    return True


if __name__ == "__main__":
    main()
