"""In-tree build of libabyssb200.so (hand-written sm_90a CUDA for the H100 behind the C ABI in include/abyss_b200.h).

    python -m abyss_b200.build [--force]

nvcc cross-compiles for sm_90a without a GPU; the .so and the host programs are git-ignored build products under
abyss_b200/lib/.
"""
from __future__ import annotations

import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "csrc")
LIBDIR = os.path.join(ROOT, "lib")
LIB = os.path.join(LIBDIR, "libabyssb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# translation unit -> the headers it includes (abb_assemble.cu takes minutes: rebuild it only when its own headers change)
SOURCES = {
    "abb_api.cu": ["abb_common.h", "abb_device.cuh", "abb_insert.cuh", "abb_shard.cuh", "abb_graph.cuh", "../../include/abyss_b200.h"],
    "abb_assemble.cu": ["abb_common.h", "abb_device.cuh", "abb_walk.cuh", "../../include/abyss_b200.h"],
    "abb_overlap.cu": ["abb_common.h", "abb_device.cuh", "abb_overlap.cuh", "../../include/abyss_b200.h"],
    "abb_konnector.cu": ["abb_common.h", "abb_device.cuh", "abb_konnector.cuh", "abb_walk.cuh", "../../include/abyss_b200.h"],
}
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [
    *ARCH, "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function", "--expt-relaxed-constexpr", "-ccbin", "g++",
]
OBJDIR = os.path.join(LIBDIR, "obj")
# the C++ host programs: the reference's command lines over the C ABI
CLIS = (("abyss-bloom-dbg", "abyss_bloom_dbg.cc"), ("abyss-bloom", "abyss_bloom.cc"), ("AdjList", "adjlist.cc"))


def _digest(paths) -> str:
    import hashlib
    h = hashlib.sha1(" ".join(FLAGS).encode())  # a change of target architecture or flags rebuilds everything
    for p in sorted(paths):
        if os.path.exists(p):
            h.update(os.path.basename(p).encode())
            h.update(open(p, "rb").read())
    return h.hexdigest()


def _stale(target: str, deps) -> bool:
    """content based (file times do not survive the snapshot that ships the tree to the GPU box): the digest of the
    dependencies is stored next to the target when it is built"""
    stamp = target + ".stamp"
    if not os.path.exists(target) or not os.path.exists(stamp):
        return True
    return open(stamp).read().strip() != _digest(deps)


def _mark(target: str, deps, digest: str | None = None) -> None:
    with open(target + ".stamp", "w") as f:
        f.write(digest or _digest(deps))


def _host_sources():
    out = []
    for d, _, fs in os.walk(os.path.join(ROOT, "host")):
        out += [os.path.join(d, f) for f in fs if f.endswith((".cc", ".h"))]
    out.append(os.path.join(ROOT, "..", "include", "abyss_b200.h"))
    return out


def _objects():
    return {src: (os.path.join(OBJDIR, src[:-3] + ".o"), [os.path.join(CSRC, src)] + [os.path.join(CSRC, h) for h in hs])
            for src, hs in SOURCES.items()}


def needs_build() -> bool:
    if os.environ.get("ABB_NO_BUILD") and os.path.exists(LIB):
        return False
    if any(_stale(o, deps) for o, deps in _objects().values()):
        return True
    if _stale(LIB, [o for o, _ in _objects().values()]):
        return True
    return any(_stale(os.path.join(LIBDIR, exe), _host_sources() + [LIB]) for exe, _ in CLIS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(OBJDIR, exist_ok=True)
    procs = []
    for src, (obj, deps) in _objects().items():
        if force or _stale(obj, deps):
            digest = _digest(deps)  # of what the compiler is about to read (an edit during the build must not look built)
            cmd = [NVCC, *FLAGS, *(["-Xptxas", "-v"] if verbose else []), "-c", "-o", obj, os.path.join(CSRC, src)]
            procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), obj, deps, digest))
    for cmd, pr, obj, deps, digest in procs:
        out, _ = pr.communicate()
        if pr.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + out)
        _mark(obj, deps, digest)
        if verbose:
            print(out)
    objs = [o for o, _ in _objects().values()]
    if force or _stale(LIB, objs):
        cmd = [NVCC, *ARCH, "-shared", "-cudart", "static", "-Xcompiler", "-fPIC", "-o", LIB, *objs,
               "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        _mark(LIB, objs)
    build_cli()
    return LIB


def build_cli() -> None:
    """the C++ host programs (abyss-bloom-dbg, abyss-bloom) that link the C-ABI library"""
    host = os.path.join(ROOT, "host")
    for exe, src in CLIS:
        cmd = ["g++", "-std=c++17", "-O2", "-Wall", "-pthread", "-o", os.path.join(LIBDIR, exe), os.path.join(host, src),
               "-L" + LIBDIR, "-labyssb200", "-Wl,-rpath,$ORIGIN"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("g++ failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        _mark(os.path.join(LIBDIR, exe), _host_sources() + [LIB])


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
