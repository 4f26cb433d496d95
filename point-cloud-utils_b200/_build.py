"""In-tree build of the native code: libpcu_b200.so (CUDA kernels + C ABI, sm_90a only, i.e. H100) and the
pybind11 module _pcu_internal that sits on top of it.  Every csrc/*.cu compiles to its own object, in parallel, and the
objects link into the library.  nvcc writes each object's dependencies (-MD) next to it, and an object is rebuilt only
when a file it was compiled from has changed since.

    python -m pcu_b200._build          # or:  import __graft_entry__; __graft_entry__.build()

nvcc cross-compiles for sm_90a without a GPU.  The artefacts stay next to the package (they are
git-ignored), so the package imports from the repository tree.
"""
import concurrent.futures
import os
import subprocess
import sys
import sysconfig

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
ROOT = os.path.dirname(PKG_DIR)
LIB = os.path.join(PKG_DIR, "libpcu_b200.so")
EXT = os.path.join(PKG_DIR, "_pcu_internal" + sysconfig.get_config_var("EXT_SUFFIX"))
OBJ_DIR = os.path.join(PKG_DIR, "build")
HOST_CXX = "/usr/bin/g++"  # the image exports CXX=/opt/gcc/bin/g++, a wrapper that lacks parts of the toolchain

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--compiler-bindir", HOST_CXX,
    "-Xcompiler", "-fPIC",
]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _depends(depfile):
    """The files a make-style dependency file lists after its target, or None when it is missing.  The units compile
    from csrc/, so the library's own files are listed relative to it and the tree can move without a rebuild."""
    try:
        with open(depfile) as fh:
            text = fh.read()
    except FileNotFoundError:
        return None
    text = text.replace("\\\n", " ").replace("\\ ", "\0")
    return [os.path.join(CSRC, w.replace("\0", " ")) for w in text.split(":", 1)[1].split()] if ":" in text else []


def _stale(obj, depfile):
    """An object is out of date when it or its dependency file is missing, or when a file it depends on is newer."""
    deps = _depends(depfile)
    return deps is None or not all(os.path.exists(d) for d in deps) or not _newer(obj, deps)


def _run(cmd, cwd=None):
    proc = subprocess.run(cmd, capture_output=True, text=True, cwd=cwd)
    if proc.returncode != 0:
        raise RuntimeError("build step failed:\n  %s\n%s%s" % (" ".join(cmd), proc.stdout, proc.stderr))
    return proc.stdout + proc.stderr


def nvcc_path():
    cand = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    return cand if os.path.exists(cand) else "nvcc"


def build(force=False, verbose=False):
    """Compile whatever is out of date.  Returns the list of artefacts."""
    import pybind11

    units = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cu")]
    os.makedirs(OBJ_DIR, exist_ok=True)
    objs = [os.path.join(OBJ_DIR, os.path.basename(u)[:-3] + ".o") for u in units]
    stale = [(u, o, o[:-2] + ".d") for u, o in zip(units, objs) if force or _stale(o, o[:-2] + ".d")]
    ptxas = ["-Xptxas", "-v"] if verbose else []
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, min(len(stale), os.cpu_count() or 1))) as pool:
        logs = list(pool.map(lambda uod: _run([nvcc_path()] + NVCC_FLAGS + ptxas + ["-MD", "-MF", uod[2], "-c", "-o", uod[1],
                                                                                   os.path.basename(uod[0])], cwd=CSRC), stale))
    if verbose:
        for log in logs:
            print(log)
    if force or not _newer(LIB, objs):
        _run([nvcc_path()] + NVCC_FLAGS + ["-shared", "-o", LIB] + objs)
    bind_src = [os.path.join(CSRC, "binding.cpp"), os.path.join(ROOT, "include", "pcu_b200.h")]
    if force or not _newer(EXT, bind_src + [LIB]):
        cmd = [HOST_CXX, "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden",
               "-I" + pybind11.get_include(), "-I" + sysconfig.get_paths()["include"],
               os.path.join(CSRC, "binding.cpp"), "-o", EXT,
               "-L" + PKG_DIR, "-lpcu_b200", "-Wl,-rpath,$ORIGIN"]
        _run(cmd)
    return [LIB, EXT]


if __name__ == "__main__":
    for path in build(force="--force" in sys.argv, verbose="-v" in sys.argv):
        print(path)
