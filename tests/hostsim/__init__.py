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
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "obm_quote.h"),
            os.path.join(_ROOT, "operator-builder_b200", "csrc", "go_unicode_tables.h"),
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
        L.hs_warp_batch_report.restype = ctypes.c_uint64
        L.hs_warp_batch_report.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_uint64,
                                           ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64,
                                           ctypes.POINTER(ctypes.c_uint64)]
        L.hs_warp_line_stats.argtypes = [ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]
        L.hs_fast_lines.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p,
                                    ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p,
                                    ctypes.c_void_p]
        L.hs_warp_units.restype = ctypes.c_uint64
        L.hs_warp_units.argtypes = [ctypes.c_void_p, ctypes.c_uint32]
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
        L.hs_classify.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p]
        L.hs_go_quote.restype = ctypes.c_uint64
        L.hs_go_quote.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64]
        u8pp = ctypes.POINTER(ctypes.POINTER(ctypes.c_uint8))
        L.hs_lex_decode_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, u8pp, ctypes.POINTER(ctypes.c_uint64),
                                          ctypes.c_void_p, ctypes.c_void_p]
        L.hs_decode_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, u8pp,
                                      ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p]
        # the parser (obm_parse.cpp) over the host tables, with registries of this library's own
        L.obm_registry_new.restype = ctypes.c_void_p
        L.obm_registry_free.argtypes = [ctypes.c_void_p]
        L.obm_registry_add.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_char_p), ctypes.c_uint32]
        L.obm_registry_define.argtypes = [ctypes.c_void_p, ctypes.c_int]
        L.obm_parse_doc.restype = ctypes.c_int64
        L.obm_parse_doc.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64, u8pp,
                                    ctypes.POINTER(ctypes.c_uint64)]
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


def classify(cps):
    """int32 code points -> uint8 bits of the product's host classes: 1 is_letter, 2 is_number, 4 is_space, 8 go_is_print"""
    cps = np.ascontiguousarray(cps, dtype=np.int32)
    out = np.zeros(len(cps), dtype=np.uint8)
    lib().hs_classify(cps.ctypes.data, len(cps), out.ctypes.data)
    return out


def go_quote(b: bytes) -> bytes:
    """the product's strconv.Quote (csrc/obm_quote.h)"""
    L = lib()
    n = L.hs_go_quote(b, len(b), None, 0)
    out = ctypes.create_string_buffer(n)
    L.hs_go_quote(b, len(b), out, n)
    return out.raw


def _take(out, outlen):
    data = ctypes.string_at(out, outlen.value)
    lib().obm_free(out)
    return data


def lex_decode_batch(data, doc_off):
    """host exact lexer + obm_decode_doc over a packed batch -> (stream bytes, stream_off uint64[ndocs+1], lexemes
    uint64[ndocs]), the layout of oracle.lex_batch_raw"""
    L = lib()
    doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
    ndocs = len(doc_off) - 1
    out, outlen = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_uint64()
    soff, nlex = np.zeros(ndocs + 1, dtype=np.uint64), np.zeros(ndocs, dtype=np.uint64)
    assert L.hs_lex_decode_batch(data.ctypes.data, doc_off.ctypes.data, ndocs, ctypes.byref(out), ctypes.byref(outlen),
                                 soff.ctypes.data, nlex.ctypes.data) == 0
    return _take(out, outlen), soff, nlex


def decode_batch(data, doc_off, tuples, tuple_off):
    """obm_decode_doc of every document of a batch from its tuples -> (stream bytes, stream_off uint64[ndocs+1])"""
    L = lib()
    doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
    tuples = np.ascontiguousarray(tuples, dtype=np.uint64)
    tuple_off = np.ascontiguousarray(tuple_off, dtype=np.uint64)
    ndocs = len(doc_off) - 1
    out, outlen = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_uint64()
    soff = np.zeros(ndocs + 1, dtype=np.uint64)
    assert L.hs_decode_batch(data.ctypes.data, doc_off.ctypes.data, ndocs, tuples.ctypes.data, tuple_off.ctypes.data,
                             ctypes.byref(out), ctypes.byref(outlen), soff.ctypes.data) == 0
    return _take(out, outlen), soff


class Registry:
    """an obm_registry of this library (names only: {marker: [args]}, or typed: define=[marker types])"""

    def __init__(self, markers=None, define=()):
        self._L = lib()
        self.handle = self._L.obm_registry_new()
        for name, args in (markers or {}).items():
            arr = (ctypes.c_char_p * max(1, len(args)))(*args)
            self._L.obm_registry_add(self.handle, name, arr, len(args))
        for t in define:
            assert self._L.obm_registry_define(self.handle, t) == 0

    def __del__(self):
        self._L.obm_registry_free(self.handle)


def parse_doc(registry, doc: bytes) -> bytes:
    """obm_parse_doc over the host exact lexer's tuples of one document -> serialised Results"""
    L = lib()
    t = lex_doc(doc)
    out, outlen = ctypes.POINTER(ctypes.c_uint8)(), ctypes.c_uint64()
    assert L.obm_parse_doc(registry.handle, doc, len(doc), t.ctypes.data, len(t), ctypes.byref(out), ctypes.byref(outlen)) >= 0
    return _take(out, outlen)


def fmt_tuples(tuples):
    names = {1: "Comment", 2: "MarkerStart", 3: "Scope", 4: "Separator", 5: "Arg", 6: "ArgAssignment", 7: "ArgDelimiter",
             8: "String", 9: "Float", 10: "Int", 11: "SynBool", 12: "Bool", 13: "Quote", 18: "MarkerEnd", 20: "EOF",
             21: "PART", 22: "FLUSH", 23: "DRIFT", 24: "LINE", 25: "LINEHI", 26: "WARN_NOSCOPE", 27: "WARN_INVALID",
             28: "ERR_MALFORMED", 29: "ERR_UNMATCHED", 30: "ERR_FLOAT", 31: "ERR_INT"}
    return [(names.get(int(t) >> 59, int(t) >> 59), int(t) & 0xFFFFFFFF, (int(t) >> 32) & 0x7FFFFFF) for t in tuples]


BAD_STARTS = (1 << 64) - 1  # hs_warp_batch*: a unit's document starts differed from doc_off


def _place(docs, skew):
    """the batch at address 16k + skew inside a poisoned buffer (readable around it, like the device buffer contract)
    -> (buffer, batch view, doc_off, output capacity)"""
    payload = b"".join(docs)
    buf = np.full(len(payload) + 96, 0x2B, dtype=np.uint8)
    start = (-buf.ctypes.data) % 16 + 16 + (skew & 15)
    buf[start:start + len(payload)] = np.frombuffer(payload, dtype=np.uint8)
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    if docs:
        off[1:] = np.cumsum([len(d) for d in docs])
    return buf, buf[start:], off, 2 * int(off[-1]) + 2 * len(docs) + 16


def tile_batch(docs, skew=0, pipeline=False):
    """Emulation of the device fast paths (pipeline=0 r01 fused tile kernel, 1 r01 two-stage pipeline, 2 the fused warp
    kernel of mode 0, run by 32 fibers per warp) over a list of documents
    -> (tuples, doc_tuple_off, stats)."""
    L = lib()
    _buf, data, off, cap = _place(docs, skew)
    out = np.zeros(cap, dtype=np.uint64)
    toff = np.zeros(len(docs) + 1, dtype=np.uint64)
    stats = np.zeros(4, dtype=np.uint64)
    fn = {0: L.hs_tile_batch, 1: L.hs_pipe_batch, 2: L.hs_warp_batch}[int(pipeline)]
    n = fn(data.ctypes.data, off.ctypes.data, len(docs), out.ctypes.data, cap, toff.ctypes.data, skew, stats.ctypes.data)
    assert n != BAD_STARTS, "the warp replay's document starts differ from doc_off"
    assert n <= cap
    return out[:n].copy(), toff, stats


# one row per unit of warp_batch's report
WARP_REPORT = np.dtype([(f, np.uint32) for f in ("u", "da", "nd", "extra", "needs_text", "paged", "deferred", "over_fin",
                                                  "long_line", "prestaged")])


def warp_batch(docs, skew=0):
    """The fused warp kernel's software pipeline replayed in k_warp_scan's order (hs_warp_batch_report), with the next
    unit's text staged over the dead text as early as the kernel stages it -> (tuples, doc_tuple_off, stats, report):
    report[u] says how unit u went (nd, extra, needs_text, paged, deferred write, more than FIN_CAP tuples, long_line,
    and whether its text was prestaged)"""
    L = lib()
    _buf, data, off, cap = _place(docs, skew)
    out = np.zeros(cap, dtype=np.uint64)
    toff = np.zeros(len(docs) + 1, dtype=np.uint64)
    stats = np.zeros(4, dtype=np.uint64)
    rcap = warp_units(off)
    report = np.zeros(rcap, dtype=WARP_REPORT)
    nu = ctypes.c_uint64()
    n = L.hs_warp_batch_report(data.ctypes.data, off.ctypes.data, len(docs), out.ctypes.data, cap, toff.ctypes.data,
                               stats.ctypes.data, report.ctypes.data, rcap, ctypes.byref(nu))
    assert n != BAD_STARTS, "the warp replay's document starts differ from doc_off"
    assert n <= cap and nu.value == rcap
    return out[:n].copy(), toff, stats, report


def warp_line_stats():
    """(marker lines the fused warp kernel's phase C stepper took, lines it handed to the generic lexer) over every
    hs_warp_batch* call of this process so far"""
    fast, generic = ctypes.c_uint64(), ctypes.c_uint64()
    lib().hs_warp_line_stats(ctypes.byref(fast), ctypes.byref(generic))
    return fast.value, generic.value


# one row per document of fast_lines
FAST_LINES = np.dtype([(f, np.uint32) for f in ("res", "lines", "ok", "ovf", "max_tuples", "max_len")])
FLR_OK, FLR_FALLBACK, FLR_NONE = 0, 1, 2


def fast_lines(data, doc_off, skews):
    """The phase C stepper (obmw::fast_line) on every marker line of each document of a packed batch, the document copied
    to skews[d] bytes past a 16-byte boundary (hs_fast_lines) -> (info, direct, toff, staged, soff): info[d] (FAST_LINES)
    says how document d went; direct[toff[d]:toff[d+1]] are its tuples with EOF (DirectSink), empty when a line was handed
    to the generic lexer; staged[soff[d]:soff[d+1]] the same from the PackSink, empty also when a line overflowed it"""
    L = lib()
    data = np.ascontiguousarray(data, dtype=np.uint8)
    off = np.ascontiguousarray(doc_off, dtype=np.uint64)
    skews = np.ascontiguousarray(skews, dtype=np.uint8)
    ndocs = len(off) - 1
    assert len(skews) == ndocs
    cap = 2 * int(off[-1]) + 4 * ndocs + 16
    direct, staged = np.zeros(cap, dtype=np.uint64), np.zeros(cap, dtype=np.uint64)
    toff, soff = np.zeros(ndocs + 1, dtype=np.uint64), np.zeros(ndocs + 1, dtype=np.uint64)
    info = np.zeros(ndocs, dtype=FAST_LINES)
    rc = L.hs_fast_lines(data.ctypes.data, off.ctypes.data, ndocs, skews.ctypes.data, direct.ctypes.data, cap, toff.ctypes.data,
                         staged.ctypes.data, cap, soff.ctypes.data, info.ctypes.data)
    assert rc == 0, rc
    return info, direct[:int(toff[-1])], toff, staged[:int(soff[-1])], soff


def warp_units(doc_off):
    """number of units the fused warp kernel cuts the batch into (make_wrec over its tiles)"""
    off = np.ascontiguousarray(doc_off, dtype=np.uint64)
    return int(lib().hs_warp_units(off.ctypes.data, len(off) - 1))
