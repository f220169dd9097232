"""TEST INFRASTRUCTURE: host build of the collection variant of the fused warp kernel (see collection.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = None


def build(force=False):
    so = os.path.join(_HERE, "libhostsim_collection.so")
    csrc = os.path.join(_ROOT, "operator-builder_b200", "csrc")
    srcs = [os.path.join(_HERE, "collection.cpp"), os.path.join(_HERE, "warp_emu.h"), os.path.join(_ROOT, "include", "obmarkers.h")]
    srcs += [os.path.join(csrc, f) for f in ("obm_core.h", "obm_pipe.h", "obm_parse_dev.h", "obm_warp.h", "obm_warp_core.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas", "-shared", "-o", so, srcs[0]])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        L.hs_warp_collection_batch.restype = ctypes.c_uint64
        L.hs_warp_collection_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p,
                                               ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p]
        _LIB = L
    return _LIB


def collection_batch(docs, skew=0, poison=0x2B):
    """The collection variant of the fused warp kernel (compute_unit<true> + write_text, 32 fibers per warp) over a list of
    documents -> (rewritten bytes, out_doc_off, tuples, doc_tuple_off, stats).  The output byte buffer is prefilled with 0xEE."""
    L = lib()
    payload = b"".join(docs)
    buf = np.full(len(payload) + 96, poison, dtype=np.uint8)
    start = (-buf.ctypes.data) % 16 + 16 + (skew & 15)
    buf[start:start + len(payload)] = np.frombuffer(payload, dtype=np.uint8)
    data = buf[start:]
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    if docs:
        off[1:] = np.cumsum([len(d) for d in docs])
    obuf = np.full(len(payload) + 96, 0xEE, dtype=np.uint8)
    ostart = (-obuf.ctypes.data) % 16
    out_bytes = obuf[ostart:]
    out_off = np.zeros(len(docs) + 1, dtype=np.uint64)
    cap = 2 * int(off[-1]) + 2 * len(docs) + 16
    out = np.zeros(cap, dtype=np.uint64)
    toff = np.zeros(len(docs) + 1, dtype=np.uint64)
    stats = np.zeros(4, dtype=np.uint64)
    n = L.hs_warp_collection_batch(data.ctypes.data, off.ctypes.data, len(docs), out_bytes.ctypes.data, out_off.ctypes.data,
                                   out.ctypes.data, cap, toff.ctypes.data, stats.ctypes.data)
    assert n <= cap
    return out_bytes[:len(payload) + 16].tobytes(), out_off, out[:n].copy(), toff, stats
