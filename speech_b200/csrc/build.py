"""Build libspeech_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m speech_b200.csrc.build [--force] [--verbose]

The library is a plain shared object (no torch / pybind dependency); Python binds it with ctypes
(speech_b200/_lib.py).  Objects are cached per source file on (mtime, flags).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(os.path.dirname(HERE), "libspeech_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-I", os.path.join(ROOT, "include"),
]


def sources():
    return sorted(f for f in os.listdir(HERE) if f.endswith(".cu"))


def _stamp(path):
    h = hashlib.sha1()
    h.update(" ".join(FLAGS).encode())
    with open(path, "rb") as fh:
        h.update(fh.read())
    for hdr in sorted(os.listdir(HERE)):
        if hdr.endswith(".cuh"):
            with open(os.path.join(HERE, hdr), "rb") as fh:
                h.update(fh.read())
    with open(os.path.join(ROOT, "include", "speech_b200.h"), "rb") as fh:
        h.update(fh.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    objs = []
    procs = []
    for src in sources():
        sp = os.path.join(HERE, src)
        obj = os.path.join(BUILD, src[:-3] + ".o")
        stamp_file = obj + ".stamp"
        stamp = _stamp(sp)
        objs.append(obj)
        if (not force and os.path.exists(obj) and os.path.exists(stamp_file)
                and open(stamp_file).read() == stamp):
            continue
        cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", sp, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, stamp_file, stamp, subprocess.Popen(
            cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, stamp_file, stamp, pr in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            failed = True
            sys.stderr.write("nvcc failed for %s:\n%s\n" % (src, out))
        else:
            if verbose or "warning" in out:
                sys.stderr.write(out)
            with open(stamp_file, "w") as fh:
                fh.write(stamp)
    if failed:
        raise RuntimeError("speech_b200: CUDA build failed")
    newest = max(os.path.getmtime(o) for o in objs)
    if force or procs or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC] + FLAGS[:2] + ["-shared", "-o", LIB] + objs + ["-lcudart"]
        subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
