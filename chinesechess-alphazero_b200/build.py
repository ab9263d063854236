"""Build recipe for the native code of cczero-b200.

`build_cuda()`  -> chinesechess-alphazero_b200/libcczero_b200.so   (nvcc, sm_90a; THE product)
`build_emul()`  -> tests/simt_emul/libcz_emul.so                   (g++ -DCZ_EMUL; test tier only)

Both are built in-tree so the .so travels with the repo snapshot to the GPU box.
nvcc cross-compiles sm_90a without a GPU.
"""
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
CUDA_LIB = os.path.join(HERE, "libcczero_b200.so")
EMUL_LIB = os.path.join(ROOT, "tests", "simt_emul", "libcz_emul.so")

# translation units: (file, extra nvcc flags)
#   integer / tree code is compiled with -fmad=false so that fp64 PUCT arithmetic rounds exactly
#   like the reference's Python floats (no contraction of a*b+c into fma).
INT_UNITS = ["cz_env_api.cu", "cz_tree_api.cu", "cz_replay.cu"]
NN_UNITS = ["cz_nn.cu", "cz_train.cu"]
HOST_UNITS = ["cz_err.cpp"]

NVCC_COMMON = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
               "-Xcompiler", "-fPIC", "-I", os.path.join(ROOT, "include")]


def _existing(units):
    return [u for u in units if os.path.exists(os.path.join(CSRC, u))]


def _stamp(files, flags):
    h = hashlib.sha256()
    for f in sorted(files):
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(repr(flags).encode())
    return h.hexdigest()


def _sources_and_headers():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC) if os.path.isfile(os.path.join(CSRC, f))] + [os.path.join(ROOT, "include", "cczero_b200.h")]


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + "\n")
        raise RuntimeError("build failed: " + cmd[0])
    return r.stdout


def build_cuda(force=False, verbose=False):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    stamp_file = CUDA_LIB + ".stamp"
    stamp = _stamp(_sources_and_headers(), NVCC_COMMON)
    if not force and os.path.exists(CUDA_LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return CUDA_LIB
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    objs = []
    jobs = []
    for u in _existing(INT_UNITS):
        o = os.path.join(objdir, u + ".o")
        jobs.append([nvcc] + NVCC_COMMON + ["-fmad=false", "-c", os.path.join(CSRC, u), "-o", o])
        objs.append(o)
    for u in _existing(NN_UNITS):
        o = os.path.join(objdir, u + ".o")
        jobs.append([nvcc] + NVCC_COMMON + ["-c", os.path.join(CSRC, u), "-o", o])
        objs.append(o)
    for u in _existing(HOST_UNITS):
        o = os.path.join(objdir, u + ".o")
        jobs.append([nvcc] + NVCC_COMMON + ["-c", os.path.join(CSRC, u), "-o", o])
        objs.append(o)
    procs = [subprocess.Popen(j, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True) for j in jobs]
    for j, p in zip(jobs, procs):
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(" ".join(j) + "\n" + out + "\n")
            raise RuntimeError("nvcc failed")
        if verbose and out.strip():
            print(out)
    _run([nvcc, "-shared", "-Xlinker", "-Bsymbolic", "-o", CUDA_LIB] + objs + ["-lcudart", "-ldl"])
    with open(stamp_file, "w") as f:
        f.write(stamp)
    return CUDA_LIB


def build_emul(force=False):
    """CPU SIMT-emulation build of the integer kernels.  Test infrastructure only."""
    srcs = [os.path.join(CSRC, u) for u in _existing(INT_UNITS)]
    host = [os.path.join(CSRC, u) for u in _existing(HOST_UNITS)]
    emul = os.path.join(ROOT, "tests", "simt_emul", "simt_emul.cpp")
    flags = ["-std=c++17", "-O2", "-g", "-DCZ_EMUL", "-ffp-contract=off", "-fPIC", "-shared",
             "-I", os.path.join(ROOT, "include")]
    stamp_file = EMUL_LIB + ".stamp"
    stamp = _stamp(_sources_and_headers() + [emul], flags)
    if not force and os.path.exists(EMUL_LIB) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return EMUL_LIB
    cmd = ["g++"] + flags
    for s in srcs:
        cmd += ["-x", "c++", s]
    for s in host + [emul]:
        cmd += ["-x", "c++", s]
    cmd += ["-Wl,-Bsymbolic", "-o", EMUL_LIB, "-lpthread"]
    _run(cmd)
    with open(stamp_file, "w") as f:
        f.write(stamp)
    return EMUL_LIB


if __name__ == "__main__":
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    if which in ("cuda", "all"):
        print(build_cuda(force="--force" in sys.argv, verbose=True))
    if which in ("emul", "all"):
        print(build_emul(force="--force" in sys.argv))
