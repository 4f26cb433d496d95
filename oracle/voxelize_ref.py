"""The reference's triangle-box test behind voxelize_triangle_mesh's candidate loop (ref_voxelize_shim.cpp), for the
tests of tests/test_voxelize_triangle_mesh.py.

build() compiles oracle/_ref/libpcu_ref_voxelize.so (git-ignored) where a checkout of the reference is present, with
the flags of the reference's x86 wheel (-O3 -msse3 -ffp-contract=off) and the system compiler the other oracle builds
pin; elsewhere it keeps a prebuilt library, if any, and does nothing else.  REF_DIR overrides the reference's
location, as it does for oracle/Makefile."""
import ctypes
import os
import subprocess

import numpy as np

from oracle import oracle as O

_HERE = os.path.dirname(os.path.abspath(__file__))
_SRC = os.path.join(_HERE, "ref_voxelize_shim.cpp")
_LIB = os.path.join(_HERE, "_ref", "libpcu_ref_voxelize.so")
_CXX = "/usr/bin/g++"
_fn = None


def _ref_dir():
    return os.environ.get("REF_DIR", "/root/reference")


def build():
    """Compiles the shim when the reference's tribox.h is present and the library is missing or older than the shim."""
    tribox = os.path.join(_ref_dir(), "src", "common", "tribox.h")
    if not os.path.exists(tribox):
        return
    if os.path.exists(_LIB) and os.path.getmtime(_LIB) >= os.path.getmtime(_SRC):
        return
    os.makedirs(os.path.dirname(_LIB), exist_ok=True)
    cmd = [_CXX, "-O3", "-msse3", "-ffp-contract=off", "-std=c++17", "-fPIC", "-shared",
           "-I" + os.path.join(_ref_dir(), "src"), "-o", _LIB, _SRC]
    out = subprocess.run(cmd, capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("voxelize oracle build failed:\n" + out.stdout + out.stderr)


def available():
    return os.path.exists(_LIB)


def _lib():
    global _fn
    if _fn is None:
        fn = ctypes.CDLL(_LIB).pcu_ref_voxelize
        fn.restype = ctypes.c_int64
        fn.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p,
                       ctypes.c_int, ctypes.c_void_p, ctypes.c_int64]
        _fn = fn
    return _fn


def voxelize_triangle_mesh(v, f, voxel_size, voxel_origin, full_x=True):
    """The reference's triBoxOverlap over each face's candidates, then the reference wrapper's
    morton_decode(np.unique(morton_encode(ijk))).  full_x=False: the reference's own x loop, [inix, inix];
    full_x=True: x over [inix, inox].  v is widened to fp64, f must index v; voxel_size and voxel_origin are 3-vectors."""
    fn = _lib()
    v = np.ascontiguousarray(v, dtype=np.float64)
    f = np.ascontiguousarray(f, dtype=np.int64)
    size = np.ascontiguousarray(voxel_size, dtype=np.float64)
    origin = np.ascontiguousarray(voxel_origin, dtype=np.float64)
    cap = 64 * f.shape[0] + 64
    while True:
        out = np.empty((cap, 3), np.int32)
        n = fn(v.ctypes.data, v.shape[0], f.ctypes.data, f.shape[0], origin.ctypes.data, size.ctypes.data, int(bool(full_x)),
               out.ctypes.data, cap)
        if n <= cap:
            break
        cap = int(n)
    return O.morton_decode(np.unique(O.morton_encode(out[:n])))
