"""oracle/build_ref.py -- TEST INFRASTRUCTURE.

Compiles the reference's four CUDA extensions UNMODIFIED, from the sources where they lie under
$GFPP_REFERENCE_ROOT, for sm_90a, into oracle/_ref/ (git-ignored).  No reference source is copied into this repository.

Recipe (SURVEY.md appendix A): torch.utils.cpp_extension.load with the flags of the reference's own backend.py
(modules/radnerfs/raymarching/backend.py:6-9 etc.), the only change being -std=c++17 instead of -std=c++14
(torch 2.11 headers require it), TORCH_CUDA_ARCH_LIST=9.0a, build directory outside the read-only tree.

On a GPU these modules are the SECOND oracle: the reference's own kernels, which pin oracle/native_ops.c
op by op (tests/test_gpu_ref_pin.py) and serve as the "kernel to beat" GPU baseline in bench.py.
"""
import os
import sys
import time

REF = os.environ.get("GFPP_REFERENCE_ROOT", "/root/reference")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "_ref")
ARCH = "9.0a"

EXTS = {
    "_raymarching_face": ("modules/radnerfs/raymarching/src", ["raymarching.cu", "bindings.cpp"]),
    "_gridencoder": ("modules/radnerfs/encoders/gridencoder/src", ["gridencoder.cu", "bindings.cpp"]),
    "_shencoder": ("modules/radnerfs/encoders/shencoder/src", ["shencoder.cu", "bindings.cpp"]),
    "_freqencoder": ("modules/radnerfs/encoders/freqencoder/src", ["freqencoder.cu", "bindings.cpp"]),
}


def main():
    if not os.path.isdir(os.path.join(REF, "modules", "radnerfs")):
        print(f"[build_ref] {REF} not present: nothing to do")
        return 0
    os.environ["TORCH_CUDA_ARCH_LIST"] = ARCH
    os.environ.setdefault("MAX_JOBS", "4")
    from torch.utils.cpp_extension import load
    nvcc_flags = ["-O3", "-std=c++17", "-U__CUDA_NO_HALF_OPERATORS__", "-U__CUDA_NO_HALF_CONVERSIONS__", "-U__CUDA_NO_HALF2_OPERATORS__"]
    for name, (sub, files) in EXTS.items():
        bdir = os.path.join(OUT, name)
        so = os.path.join(bdir, name + ".so")
        stamp = os.path.join(bdir, "arch.txt")   # a module built for another architecture does not load: rebuild it
        if os.path.exists(so) and os.path.exists(stamp) and open(stamp).read().strip() == ARCH:
            print(f"[build_ref] {name}: up to date")
            continue
        os.makedirs(bdir, exist_ok=True)
        if os.path.exists(so):
            os.unlink(so)
        t0 = time.time()
        load(name=name, sources=[os.path.join(REF, sub, f) for f in files], extra_cflags=["-O3", "-std=c++17"],
             extra_cuda_cflags=nvcc_flags, build_directory=bdir, verbose=False, is_python_module=False)
        with open(stamp, "w") as fh:
            fh.write(ARCH + "\n")
        print(f"[build_ref] {name}: built in {time.time() - t0:.0f}s -> {so}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
