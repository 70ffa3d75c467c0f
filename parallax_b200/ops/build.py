"""In-tree build of the native library (sm_90a only).

    python -m parallax_b200.ops.build            # incremental
    python -m parallax_b200.ops.build --force

Produces `parallax_b200/ops/libparallax_b200.so` (git-ignored).  Every
translation unit is compiled with ``-gencode arch=compute_90a,code=sm_90a
-lineinfo``; there is no other target.  The reference's build (`horovod/setup.py`, TF bazel with
compute 3.5/7.0 — `tensorflow/configure.py:36-39`) has no counterpart here:
one nvcc invocation per file, one link.
"""
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libparallax_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
          "-Xcompiler", "-fvisibility=default", "--expt-relaxed-constexpr"]


def nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"),
              "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


def sources():
    out = []
    for sub in ("kernels", "runtime"):
        d = os.path.join(CSRC, sub)
        for f in sorted(os.listdir(d)):
            if f.endswith((".cu", ".cpp")):
                out.append(os.path.join(d, f))
    return out


def _headers_digest():
    h = hashlib.sha1()
    for root, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".h", ".cuh", ".hpp")):
                with open(os.path.join(root, f), "rb") as fh:
                    h.update(fh.read())
    return h.hexdigest()


def _stamp(src, hdr):
    with open(src, "rb") as f:
        return hashlib.sha1(f.read() + hdr.encode() +
                            " ".join(ARCH + COMMON).encode()).hexdigest()


def _compile(src, hdr, force, verbose):
    os.makedirs(OBJ, exist_ok=True)
    base = os.path.basename(src).rsplit(".", 1)[0]
    obj = os.path.join(OBJ, base + ".o")
    stampf = obj + ".stamp"
    st = _stamp(src, hdr)
    if not force and os.path.exists(obj) and os.path.exists(stampf) and \
            open(stampf).read() == st:
        return obj, False
    cmd = [nvcc()] + ARCH + COMMON + ["-I", os.path.join(CSRC, "kernels"),
                                      "-I", os.path.join(CSRC, "runtime")]
    if src.endswith(".cpp"):
        cmd += ["-x", "cu"]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    if verbose:
        sys.stderr.write(r.stderr)
    with open(stampf, "w") as f:
        f.write(st)
    return obj, True


def build(force=False, verbose=False):
    if nvcc() is None:
        raise RuntimeError("nvcc not found; cannot build libparallax_b200.so")
    hdr = _headers_digest()
    srcs = sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, hdr, force, verbose), srcs))
    objs = [o for o, _ in res]
    changed = any(c for _, c in res)
    if changed or force or not os.path.exists(LIB):
        cmd = [nvcc()] + ARCH + ["-shared", "-o", LIB] + objs + \
            ["-lcudart", "-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(path)
