"""TEST INFRASTRUCTURE: host build of the product's lexer core + decoder (see hostsim.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(os.path.dirname(_HERE))
_LIB = None


def build(force=False):
    so = os.path.join(_HERE, "libhostsim.so")
    srcs = [os.path.join(_HERE, "hostsim.cpp"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_decode.cpp"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_parse.cpp"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_core.h"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_tile.h"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_pipe.h"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_large.h"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_warp.h"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_warp_core.h"),
            os.path.join(_HERE, "warp_emu.h"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_parse_dev.h"),
            os.path.join(_ROOT, "include", "obmarkers.h")]
    if force or not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-Wall", "-Wextra", "-Wno-unknown-pragmas", *(["-DOBMW_DEBUG"] if os.environ.get("OBMW_DEBUG") else []), "-shared", "-o", so,
                               srcs[0], srcs[1], srcs[2]])
    return so


def lib():
    global _LIB
    if _LIB is None:
        L = ctypes.CDLL(build())
        L.hs_lex_doc.restype = ctypes.c_uint64
        L.hs_lex_doc.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64,
                                 ctypes.POINTER(ctypes.c_uint32), ctypes.POINTER(ctypes.c_uint32)]
        L.hs_lex_doc_by_lines.restype = ctypes.c_uint64
        L.hs_lex_doc_by_lines.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64]
        L.hs_tile_batch.restype = ctypes.c_uint64
        L.hs_tile_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64,
                                    ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p]
        L.hs_pipe_batch.restype = ctypes.c_uint64
        L.hs_pipe_batch.argtypes = L.hs_tile_batch.argtypes
        L.hs_warp_batch.restype = ctypes.c_uint64
        L.hs_warp_batch.argtypes = L.hs_tile_batch.argtypes
        L.hs_large_doc.restype = ctypes.c_uint64
        L.hs_large_doc.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint32)]
        L.hs_large_chunk_starts.restype = ctypes.c_uint32
        L.hs_large_chunk_starts.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]
        L.hs_utf8_plain.argtypes = [ctypes.c_char_p, ctypes.c_uint32, ctypes.c_uint32]
        L.hs_parse_float_err.argtypes = [ctypes.c_char_p, ctypes.c_uint32]
        L.hs_atoi_err.argtypes = [ctypes.c_char_p, ctypes.c_uint32]
        L.obm_decode_doc.restype = ctypes.c_int64
        L.obm_decode_doc.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64,
                                     ctypes.POINTER(ctypes.POINTER(ctypes.c_uint8)), ctypes.POINTER(ctypes.c_uint64)]
        L.obm_free.argtypes = [ctypes.c_void_p]
        _LIB = L
    return _LIB


def lex_doc(doc: bytes, by_lines=False):
    """-> numpy uint64 tuple array produced by the host build of the core."""
    L = lib()
    cap = 2 * len(doc) + 16
    out = np.zeros(cap, dtype=np.uint64)
    if by_lines:
        n = L.hs_lex_doc_by_lines(doc, len(doc), out.ctypes.data, cap)
    else:
        n = L.hs_lex_doc(doc, len(doc), out.ctypes.data, cap, None, None)
    assert n <= cap
    return out[:n].copy()


def large_doc(doc: bytes):
    """chunk-parallel exact path (obm_large.h) -> (tuples, chain_validated)"""
    L = lib()
    cap = 2 * len(doc) + 16
    out = np.zeros(cap, dtype=np.uint64)
    used = ctypes.c_uint32(0)
    n = L.hs_large_doc(doc, len(doc), out.ctypes.data, cap, ctypes.byref(used))
    assert n <= cap
    return out[:n].copy(), bool(used.value)


def large_chunk_starts(doc: bytes):
    """resolved (start, line) of every chunk of the chunk-parallel path -> two numpy uint32 arrays"""
    L = lib()
    nc = max(1, -(-len(doc) // 1024))
    cs = np.zeros(nc, dtype=np.uint32)
    line = np.zeros(nc, dtype=np.uint32)
    assert L.hs_large_chunk_starts(doc, len(doc), cs.ctypes.data, line.ctypes.data) == nc
    return cs, line


def decode(doc: bytes, tuples, L=None) -> bytes:
    """tuples -> serialised lexeme stream (same record format as the oracle's)."""
    L = L or lib()
    tuples = np.ascontiguousarray(tuples, dtype=np.uint64)
    out = ctypes.POINTER(ctypes.c_uint8)()
    outlen = ctypes.c_uint64()
    n = L.obm_decode_doc(doc, len(doc), tuples.ctypes.data, len(tuples), ctypes.byref(out), ctypes.byref(outlen))
    assert n >= 0
    data = ctypes.string_at(out, outlen.value)
    L.obm_free(out)
    return data


def fmt_tuples(tuples):
    names = {1: "Comment", 2: "MarkerStart", 3: "Scope", 4: "Separator", 5: "Arg", 6: "ArgAssignment", 7: "ArgDelimiter",
             8: "String", 9: "Float", 10: "Int", 11: "SynBool", 12: "Bool", 13: "Quote", 18: "MarkerEnd", 20: "EOF",
             21: "PART", 22: "FLUSH", 23: "DRIFT", 24: "LINE", 25: "LINEHI", 26: "WARN_NOSCOPE", 27: "WARN_INVALID",
             28: "ERR_MALFORMED", 29: "ERR_UNMATCHED", 30: "ERR_FLOAT", 31: "ERR_INT"}
    return [(names.get(int(t) >> 59, int(t) >> 59), int(t) & 0xFFFFFFFF, (int(t) >> 32) & 0x7FFFFFF) for t in tuples]


def tile_batch(docs, skew=0, pipeline=False):
    """Emulation of the device fast paths (pipeline=0 r01 fused tile kernel, 1 r01 two-stage pipeline, 2 the fused warp
    kernel of mode 0, run by 32 fibers per warp) over a list of documents
    -> (tuples, doc_tuple_off, stats)."""
    L = lib()
    # the batch sits at address = 16k + skew inside a poisoned buffer (readable around it, like the device buffer contract)
    payload = b"".join(docs)
    buf = np.full(len(payload) + 96, 0x2B, dtype=np.uint8)
    start = (-buf.ctypes.data) % 16 + 16 + (skew & 15)
    buf[start:start + len(payload)] = np.frombuffer(payload, dtype=np.uint8)
    data = buf[start:]
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    if docs:
        off[1:] = np.cumsum([len(d) for d in docs])
    cap = 2 * int(off[-1]) + 2 * len(docs) + 16
    out = np.zeros(cap, dtype=np.uint64)
    toff = np.zeros(len(docs) + 1, dtype=np.uint64)
    stats = np.zeros(4, dtype=np.uint64)
    fn = {0: L.hs_tile_batch, 1: L.hs_pipe_batch, 2: L.hs_warp_batch}[int(pipeline)]
    n = fn(data.ctypes.data, off.ctypes.data, len(docs), out.ctypes.data, cap, toff.ctypes.data, skew, stats.ctypes.data)
    assert n <= cap
    return out[:n].copy(), toff, stats
