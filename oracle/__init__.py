"""CPU oracle loader (TEST INFRASTRUCTURE ONLY).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this package.  The product package never does.  See oracle/lexer_oracle.c for what the
oracle restates (reference: internal/markers/lexer/*.go) and how it is pinned.
"""
import ctypes
import os
import struct
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

LEXEME_NAMES = ["Error", "Comment", "MarkerStart", "Scope", "Separator", "Arg", "ArgAssignment", "ArgDelimiter",
                "StringLiteral", "FloatLiteral", "IntegerLiteral", "SyntheticBoolLiteral", "BoolLiteral", "Quote",
                "SliceBegin", "SliceEnd", "SliceDelimiter", "NakedSliceDelimiter", "MarkerEnd", "Warning", "EOF"]


def build(force=False):
    so = os.path.join(_HERE, "liblexer_oracle.so")
    src = os.path.join(_HERE, "lexer_oracle.c")
    if force or not os.path.exists(so) or (os.path.exists(src) and os.path.getmtime(so) < os.path.getmtime(src)):
        subprocess.check_call(["make", "-C", _HERE, "-s", "CC=gcc"])
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liblexer_oracle.so")
        if not os.path.exists(so):
            build()
        L = ctypes.CDLL(so)
        u8p, u64p = ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_uint64)
        L.obo_lex.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.POINTER(u8p), u64p, u64p]
        L.obo_lex_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.POINTER(u8p), u64p,
                                    ctypes.c_void_p, ctypes.c_void_p]
        L.obo_scan_batch.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_int, u64p, u64p, u64p,
                                     ctypes.c_void_p]
        L.obo_free.argtypes = [ctypes.c_void_p]
        L.obo_prim_new.restype = ctypes.c_void_p
        L.obo_prim_new.argtypes = [ctypes.c_char_p, ctypes.c_uint64]
        for f in ("obo_prim_free", "obo_prim_consumeWhitespace"):
            getattr(L, f).argtypes = [ctypes.c_void_p]
        L.obo_prim_consume.argtypes = [ctypes.c_void_p, ctypes.c_char_p]
        L.obo_prim_consumed.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_char_p), ctypes.c_int]
        L.obo_prim_peeked.argtypes = L.obo_prim_consumed.argtypes
        L.obo_prim_consumedWhitespaced.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_char_p), ctypes.c_int]
        L.obo_prim_peekedWhitespaced.argtypes = L.obo_prim_consumedWhitespaced.argtypes
        L.obo_prim_consumeUntil.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32), ctypes.c_int]
        L.obo_prim_peek.argtypes = [ctypes.c_void_p]
        L.obo_prim_peek.restype = ctypes.c_int32
        L.obo_prim_peekN.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int32)]
        L.obo_prim_buffer.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint64]
        L.obo_prim_buffer.restype = ctypes.c_uint64
        L.obo_prim_pos.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64)]
        L.obo_parse_float_err.argtypes = [ctypes.c_char_p, ctypes.c_uint64]
        L.obo_atoi_err.argtypes = [ctypes.c_char_p, ctypes.c_uint64]
        L.obo_quote.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64]
        L.obo_quote.restype = ctypes.c_uint64
        L.obo_classify.argtypes = [ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p]
        _LIB = L
    return _LIB


def quote(b: bytes) -> bytes:
    """strconv.Quote of a byte string (Go 1.16, Unicode 13.0 IsPrint)"""
    L = lib()
    n = L.obo_quote(b, len(b), None, 0)
    out = ctypes.create_string_buffer(n)
    L.obo_quote(b, len(b), out, n)
    return out.raw


def classify(cps):
    """int32 code points -> uint8 bits: 1 unicode.IsLetter, 2 IsNumber, 4 IsSpace, 8 strconv.IsPrint"""
    import numpy as np
    cps = np.ascontiguousarray(cps, dtype=np.int32)
    out = np.zeros(len(cps), dtype=np.uint8)
    lib().obo_classify(cps.ctypes.data, len(cps), out.ctypes.data)
    return out


def generate_corpus(ndocs: int, doc_bytes: int = 4096, first_doc: int = 0, flavour: int = 0):
    """The bench corpus (csrc/obm_corpus.h) from a host library of its own (oracle/corpus_gen.cpp): the reference arm of
    bench.py must not map product code.  -> (uint8 bytes, uint64 doc_off[ndocs+1])"""
    import numpy as np
    so = os.path.join(_HERE, "libcorpus_gen.so")
    if not os.path.exists(so):
        build(force=True)
    G = ctypes.CDLL(so)
    G.obc_generate_corpus_host.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_int]
    data = np.empty(ndocs * doc_bytes, dtype=np.uint8)
    off = np.empty(ndocs + 1, dtype=np.uint64)
    rc = G.obc_generate_corpus_host(data.ctypes.data, off.ctypes.data, ndocs, doc_bytes, first_doc, flavour)
    if rc != 0:
        raise RuntimeError(f"obc_generate_corpus_host -> {rc}")
    return data, off


def parse_stream(buf):
    """Serialised stream -> list of (type, value bytes, line, col)."""
    out, i, n = [], 0, len(buf)
    while i < n:
        typ = buf[i]
        line, col, vlen = struct.unpack_from("<III", buf, i + 1)
        out.append((typ, bytes(buf[i + 13:i + 13 + vlen]), line, col))
        i += 13 + vlen
    return out


def lex_raw(doc: bytes) -> bytes:
    """Serialised lexeme stream of one document: [u8 type][u32 line][u32 col][u32 vlen][value]..."""
    L = lib()
    out = ctypes.POINTER(ctypes.c_uint8)()
    outlen, nlex = ctypes.c_uint64(), ctypes.c_uint64()
    L.obo_lex(doc, len(doc), ctypes.byref(out), ctypes.byref(outlen), ctypes.byref(nlex))
    data = ctypes.string_at(out, outlen.value)
    L.obo_free(out)
    return data


def lex(doc: bytes):
    return parse_stream(lex_raw(doc))


def lex_batch_raw(bytes_np, doc_off_np):
    """numpy uint8 bytes + uint64 doc_off[ndocs+1] -> (stream bytes, stream_off uint64[ndocs+1], lexemes uint64[ndocs])"""
    import numpy as np
    L = lib()
    ndocs = len(doc_off_np) - 1
    out = ctypes.POINTER(ctypes.c_uint8)()
    outlen = ctypes.c_uint64()
    soff = np.zeros(ndocs + 1, dtype=np.uint64)
    nlex = np.zeros(ndocs, dtype=np.uint64)
    L.obo_lex_batch(bytes_np.ctypes.data, doc_off_np.ctypes.data, ndocs, ctypes.byref(out), ctypes.byref(outlen),
                    soff.ctypes.data, nlex.ctypes.data)
    data = ctypes.string_at(out, outlen.value)
    L.obo_free(out)
    return data, soff, nlex


def scan_batch(bytes_np, doc_off_np, nthreads=1, want_doc_hash=False):
    """Count/hash-only pass used as the CPU baseline. Returns (n_lexemes, n_markers, hash[, doc_hash])."""
    import numpy as np
    L = lib()
    ndocs = len(doc_off_np) - 1
    nl, nm, h = ctypes.c_uint64(), ctypes.c_uint64(), ctypes.c_uint64()
    dh = np.zeros(ndocs, dtype=np.uint64) if want_doc_hash else None
    L.obo_scan_batch(bytes_np.ctypes.data, doc_off_np.ctypes.data, ndocs, nthreads, ctypes.byref(nl), ctypes.byref(nm),
                     ctypes.byref(h), dh.ctypes.data if want_doc_hash else None)
    return (nl.value, nm.value, h.value, dh) if want_doc_hash else (nl.value, nm.value, h.value)
