"""Build libgfpp.so (hand-written sm_90a CUDA behind the C-ABI of include/gfpp.h) IN-TREE with nvcc.

    python -m genefaceplusplus_b200.build [--force]

nvcc cross-compiles without a GPU; the resulting genefaceplusplus_b200/libgfpp.so is loaded from the package directory.
"""
import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libgfpp.so")
SOURCES = ["capi.cu", "ops_kernels.cu", "head_kernel.cu", "torso_kernel.cu", "tc_pack.cu", "head_tc_kernel.cu", "head_v2_kernel.cu", "sr_kernel.cu", "sr_train_kernel.cu", "torso_sr_kernel.cu", "train_kernels.cu", "grid_kernels.cu", "torso_grid_kernel.cu", "field_train_kernel.cu", "field_train_tc_kernel.cu", "torso_train_kernel.cu", "torso_sr_points_kernel.cu", "grid_half_kernels.cu", "torso_pass_kernels.cu", "video_kernels.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _deps():
    out = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    out.append(os.path.join(os.path.dirname(HERE), "include", "gfpp.h"))
    return out


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(p) > t for p in _deps())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJ, exist_ok=True)

    def cc(src):
        obj = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [NVCC, *FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj, r.stderr

    with cf.ThreadPoolExecutor(max_workers=4) as ex:
        results = list(ex.map(cc, SOURCES))
    if verbose:
        for _, err in results:
            sys.stderr.write(err)
    r = subprocess.run([NVCC, "-shared", "-o", LIB, *[o for o, _ in results]], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
