"""Build libxtb200.so (hand-written CUDA for the H100, sm_90a) in-tree with nvcc.

The built library lives at xingtian_b200/lib/libxtb200.so (git-ignored) and is rebuilt when a source
is newer than it.  Each source compiles to an object in its own nvcc process, all at once, and the objects are linked
into the library (whole-program device compilation: no device link).  There is no CPU fallback: importing the engine
without the library raises."""
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libxtb200.so")
SOURCES = ["xtb_engine.cu", "learners.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _stale():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    deps.append(os.path.join(HERE, "..", "include", "xtb200.h"))
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def _run(cmds, verbose):
    """Run the nvcc commands at once; raise with the output of the first that fails."""
    procs = [subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True) for cmd in cmds]
    errs = [p.communicate()[1] for p in procs]
    for cmd, p, err in zip(cmds, procs, errs):
        if verbose:
            sys.stderr.write(err)
        if p.returncode != 0:
            raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), err))


def build(force=False, verbose=False):
    """Compile every CUDA source for sm_90a (nvcc cross-compiles without a GPU)."""
    if not force and not _stale():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    compile_flags = [f for f in NVCC_FLAGS if f != "-shared"] + (["-Xptxas", "-v"] if verbose else [])
    with tempfile.TemporaryDirectory() as tmp:
        objs = [os.path.join(tmp, os.path.splitext(s)[0] + ".o") for s in SOURCES]
        _run([[nvcc] + compile_flags + ["-c", "-o", o, os.path.join(CSRC, s)] for s, o in zip(SOURCES, objs)], verbose)
        _run([[nvcc] + NVCC_FLAGS + ["-o", LIB_PATH] + objs], verbose)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
