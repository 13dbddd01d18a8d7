"""Build libcotr_b200.so (sm_90a only) in-tree with nvcc.  `python -m cotr_b200.build [--force]`.

The library is a plain C-ABI shared object (include/cotr_b200.h): no torch, no pybind.  It is built in-tree
(cotr_b200/lib/) so that the package is importable straight from the repository tree.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libcotr_b200.so")
SOURCES = ["model.cu", "gemm_simt.cu", "gemm_tc.cu", "mlp_tc.cu", "attention_simt.cu", "attention_tc.cu", "attention_weights.cu", "elementwise.cu", "preprocess.cu", "dense_post.cu", "engine_ops.cu", "peer_exchange.cu", "match.cu", "refine.cu", "first_guess.cu", "resize.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _nvcc():
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else "nvcc"


def _deps():
    files = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    files.append(os.path.join(os.path.dirname(HERE), "include", "cotr_b200.h"))
    return files


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    return any(os.path.getmtime(f) > t for f in _deps())


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    obj_dir = os.path.join(LIB_DIR, "obj")
    os.makedirs(obj_dir, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(obj_dir, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj, r.stderr

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        results = list(ex.map(compile_one, SOURCES))
    if verbose:
        for _obj, log in results:
            sys.stderr.write(log)
    cmd = [nvcc, "-shared", "-cudart", "static", "-o", LIB_PATH, *[o for o, _ in results]]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
