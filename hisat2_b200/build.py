"""Build helpers: compile the CUDA library (sm_90a) and the test-side oracle.

`build_lib()` runs nvcc on hisat2_b200/csrc and leaves hisat2_b200/libht2gpu.so
in-tree (git-ignored).  nvcc cross-compiles without a GPU.  `build_oracle()`
compiles oracle/'s C restatement and, when the reference sources are present
($HT2_REFERENCE), the unmodified reference plus the staged test data into
oracle/_ref/.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "hisat2_b200", "csrc")
LIB = os.path.join(ROOT, "hisat2_b200", "libht2gpu.so")
CLI = os.path.join(ROOT, "hisat2_b200", "hisat2-b200")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++14",
    "-Xcompiler", "-fPIC", "-cudart", "static",
]
LIB_SRCS = ["ht2_gpu.cu", "ht2_inflate.cu", "ht2_index.cpp", "ht2_host.cpp", "ht2_reads.cpp", "ht2_pipeline.cpp", "ht2_compat.cpp"]


def _newer(target, srcs):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in srcs)


def _csrc_files():
    return [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "ht2gpu.h")]


def source_hash():
    """sha1 over the library's sources: ties a profile (profiles/traffic.json) to the kernels it was taken from."""
    import hashlib
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".h", ".cu", ".cpp")):
            h.update(f.encode())
            h.update(open(os.path.join(CSRC, f), "rb").read())
    return h.hexdigest()[:16]


def build_tools():
    """tools/libsimreads.so: the synthetic read generator bench.py and the full-size tests use (test tooling)."""
    src = os.path.join(ROOT, "tools", "simreads_fast.c")
    so = os.path.join(ROOT, "tools", "libsimreads.so")
    if os.path.exists(src) and not _newer(so, [src]):
        subprocess.run(["gcc", "-O2", "-shared", "-fPIC", "-o", so, src], check=True)
    return so


def build_lib(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in LIB_SRCS]
    if not force and _newer(LIB, _csrc_files()):
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    cmd = [nvcc] + NVCC_FLAGS + ["-shared", "-o", LIB] + srcs
    if os.environ.get("HT2_NO_SPLICED"):   # diagnostic build without the spliced-alignment code (refuses spliced mode)
        cmd.insert(1, "-DHT2_DISABLE_SPLICED")
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.run(cmd, check=True, cwd=CSRC)
    return LIB


def build_cli(force=False):
    """hisat2-compatible command-line front end (host C++ over the C ABI)."""
    src = os.path.join(CSRC, "..", "cli", "hisat2_b200_main.cpp")
    src = os.path.normpath(src)
    if not os.path.exists(src):
        return None
    if not force and _newer(CLI, [src, LIB]):
        return CLI
    cmd = ["g++", "-O2", "-std=c++14", "-o", CLI, src, "-I", os.path.join(ROOT, "include"),
           "-L", os.path.dirname(LIB), "-l:libht2gpu.so", "-Wl,-rpath,$ORIGIN", "-lpthread", "-ldl", "-lrt"]
    subprocess.run(cmd, check=True)
    return CLI


def build_oracle(verbose=False):
    odir = os.path.join(ROOT, "oracle")
    out = {}
    csrc = os.path.join(odir, "ht2_oracle.c")
    if os.path.exists(csrc):
        so = os.path.join(odir, "libht2oracle.so")
        if not _newer(so, [csrc]):
            subprocess.run(["gcc", "-O2", "-std=c99", "-shared", "-fPIC", "-o", so, csrc], check=True)
        out["oracle"] = so
        exe = os.path.join(odir, "ht2_oracle")     # `ht2_oracle dump <index> <reads.fa> <no_spliced>`: the checker smoke() runs
        if not _newer(exe, [csrc]):
            subprocess.run(["gcc", "-O2", "-std=gnu99", "-DHT2_ORACLE_MAIN", "-o", exe, csrc], check=True)
        out["oracle_exe"] = exe
    ref = os.environ.get("HT2_REFERENCE", "/root/reference")
    if os.path.isdir(ref):
        subprocess.run(["make", "-s", "-j8", "REF=" + ref], check=True, cwd=odir,
                       stdout=None if verbose else subprocess.DEVNULL)
        subprocess.run(["bash", os.path.join(odir, "make_data.sh")], check=True,
                       env=dict(os.environ, REF=ref), stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
        out["ref"] = os.path.join(odir, "_ref", "hisat2-align-s")
    return out


if __name__ == "__main__":
    build_lib(force="--force" in sys.argv, verbose=True)
    build_cli()
    build_tools()
    build_oracle(verbose=True)
