"""Builds libsr3_b200.so (sm_90a only) in-tree with nvcc.  No torch involved: the library is a plain C-ABI .so."""
import hashlib
import os
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "lib", "libsr3_b200.so")
SOURCES = ["engine.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "--expt-relaxed-constexpr", "-Xptxas", "-v", "-shared", "-cudart", "static"]


def _digest():
    """sha256 over EVERY file under csrc/ (recursively) and the public header: editing any kernel source triggers a rebuild."""
    h = hashlib.sha256()
    files = []
    for d, _dirs, names in os.walk(CSRC):
        files += [os.path.join(d, n) for n in names if n.endswith((".cu", ".cuh", ".h", ".inc"))]
    files.append(os.path.join(PKG, "..", "include", "sr3_b200.h"))
    for f in sorted(files):
        h.update(os.path.relpath(f, PKG).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    stamp = LIB + ".sha256"
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    tmp = LIB + ".building"                    # the library is replaced atomically: a snapshot of the tree never sees a half-written .so
    cmd = [nvcc] + NVCC_FLAGS + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", tmp]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    log = os.path.join(PKG, "lib", "build.log")
    with open(log, "w") as fh:
        fh.write(" ".join(cmd) + "\n" + r.stdout)
    if verbose or r.returncode != 0:
        print(r.stdout)
    if r.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("nvcc failed, see " + log)
    os.replace(tmp, LIB)
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
