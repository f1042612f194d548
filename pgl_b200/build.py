"""Build libpglb.so (the C-ABI shared library, include/pglb.h) in-tree with nvcc for sm_90a.

    python pgl_b200/build.py [--force]      (run as a script: importing the package needs the library)

Also builds, when a reference checkout is present ($PGL_REFERENCE), a METIS shared library from the
reference's vendored third-party METIS 5.1.0 sources where they lie (IDXTYPEWIDTH 64) into
``pgl_b200/third_party/libmetis_i64.so`` -- a third-party dependency like cuBLAS, not
product source; nothing from it is copied into the repository.
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpglb.so")
METIS_LIB = os.path.join(HERE, "third_party", "libmetis_i64.so")
REF_METIS = os.path.join(os.environ.get("PGL_REFERENCE", "/root/reference"), "pgl", "third_party", "metis")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
    "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
]


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("command failed: %s\n%s" % (" ".join(cmd), r.stdout[-6000:]))
    return r.stdout


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cpp")))


def _deps():
    return _sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.inl")) + \
        [os.path.join(ROOT, "include", "pglb.h")]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_lib(force=False, verbose=False):
    if not force and not _stale(LIB, _deps()):
        return LIB
    bdir = os.path.join(HERE, "build")
    os.makedirs(bdir, exist_ok=True)
    objs = []
    procs = []
    hdrs = glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.inl")) + \
        [os.path.join(ROOT, "include", "pglb.h")]
    for s in _sources():
        o = os.path.join(bdir, os.path.basename(s) + ".o")
        objs.append(o)
        if not force and not _stale(o, [s] + hdrs):
            continue
        # host-only C++ (host.cpp: the alias table build) must round like the reference: no FMA contraction
        host = ["-Xcompiler", "-ffp-contract=off"] if s.endswith(".cpp") else []
        cmd = ["nvcc"] + NVCC_FLAGS + host + (["-Xptxas", "-v"] if verbose else []) + ["-c", s, "-o", o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                          text=True)))
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError("nvcc failed on %s\n%s" % (s, out[-8000:]))
        if verbose:
            print(out)
    _run(["nvcc", "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs +
         ["-lcudart", "-ldl"])
    return LIB


def build_metis(force=False, jobs=8):
    if os.path.exists(METIS_LIB) and not force:
        return METIS_LIB
    if not os.path.isdir(REF_METIS):
        return None
    os.makedirs(os.path.dirname(METIS_LIB), exist_ok=True)
    bdir = os.path.join(HERE, "build", "metis")
    os.makedirs(bdir, exist_ok=True)
    incs = ["-I" + os.path.join(REF_METIS, "include"), "-I" + os.path.join(REF_METIS, "GKlib"),
            "-I" + os.path.join(REF_METIS, "libmetis")]
    srcs = glob.glob(os.path.join(REF_METIS, "GKlib", "*.c")) + \
        glob.glob(os.path.join(REF_METIS, "libmetis", "*.c"))
    objs, procs = [], []
    for s in srcs:
        o = os.path.join(bdir, os.path.basename(os.path.dirname(s)) + "_" + os.path.basename(s)[:-2] + ".o")
        objs.append(o)
        procs.append((s, subprocess.Popen(["gcc", "-O2", "-fPIC", "-w", "-c", s, "-o", o] + incs,
                                          stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        if len(procs) >= jobs:
            s0, p0 = procs.pop(0)
            out, _ = p0.communicate()
            if p0.returncode != 0:
                raise RuntimeError("gcc failed on %s\n%s" % (s0, out[-3000:]))
    for s0, p0 in procs:
        out, _ = p0.communicate()
        if p0.returncode != 0:
            raise RuntimeError("gcc failed on %s\n%s" % (s0, out[-3000:]))
    _run(["gcc", "-shared", "-o", METIS_LIB] + objs + ["-lm"])
    return METIS_LIB


def build_all(force=False, verbose=False):
    lib = build_lib(force=force, verbose=verbose)
    metis = build_metis(force=False)
    return lib, metis


if __name__ == "__main__":
    print(build_all(force="--force" in sys.argv, verbose="-v" in sys.argv))
