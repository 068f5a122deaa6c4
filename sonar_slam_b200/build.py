"""Build libsonarfe.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m sonar_slam_b200.build [--force] [--verbose]

The shared object lands next to this file (sonar_slam_b200/libsonarfe.so); it is
git-ignored.  A rebuild happens whenever the sources, the header or the flags change.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libsonarfe.so")
STAMP = os.path.join(HERE, "build", "stamp.txt")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _fingerprint():
    h = hashlib.sha256(" ".join(FLAGS).encode())
    inc = os.path.join(os.path.dirname(HERE), "include", "sonarfe.h")
    for p in sources() + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cuh")] + [inc]:
        with open(p, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    fp = _fingerprint()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == fp:
        return LIB
    if not os.path.exists(NVCC):
        if os.path.exists(LIB):  # GPU box without sources changed: use what travelled
            return LIB
        raise RuntimeError("nvcc not found and no prebuilt libsonarfe.so")
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        procs.append((src, subprocess.Popen([NVCC] + FLAGS + ["-c", src, "-o", obj], stdout=subprocess.PIPE,
                                            stderr=subprocess.STDOUT, text=True)))
    log = []
    for src, p in procs:
        out, _ = p.communicate()
        log.append(out)
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f"nvcc failed on {src}")
    with open(os.path.join(HERE, "build", "ptxas.log"), "w") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    # hidden visibility + explicit SFE_API exports keep the ABI to what include/sonarfe.h declares
    subprocess.run([NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"],
                   check=True)
    with open(STAMP, "w") as f:
        f.write(fp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
