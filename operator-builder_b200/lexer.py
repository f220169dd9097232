"""Host-side mirror of the reference lexer's interface for this path (Python stand-in for the Go
shim in go/lexer_gpu.go, used by the tests and the bench because this image has no Go toolchain).

Reference surface (internal/markers/lexer):
    NewLexer(r io.Reader) *Lexer      lexer.go:27     -> Scanner.lex_batch(...) + Lexer(doc, tuples)
    (*Lexer).Run()                    lexer.go:43     -> Lexer.run()  (no-op: the GPU already ran)
    (*Lexer).NextLexeme() Lexeme      lexer.go:51     -> Lexer.next_lexeme()
    Lexeme{Type, Value, Pos}          lexeme.go:32-36 -> Lexeme(type, value, pos)
    LexemeType constants              lexeme.go:8-30  -> LexemeType
Errors behave like the reference: lexical errors/warnings are in-band lexemes; after the last lexeme
next_lexeme() keeps returning the zero Lexeme (Type 0, Value "") like a closed Go channel.
Infrastructure failures raise NativeError.  All scanning happens in libobmarkers.so on the GPU.
"""
import ctypes
import enum
from typing import NamedTuple

import numpy as np

from . import _native
from ._native import NativeError, ObmLexeme, ObmStats


class LexemeType(enum.IntEnum):  # lexeme.go:8-30
    Error = 0
    Comment = 1
    MarkerStart = 2
    Scope = 3
    Separator = 4
    Arg = 5
    ArgAssignment = 6
    ArgDelimiter = 7
    StringLiteral = 8
    FloatLiteral = 9
    IntegerLiteral = 10
    SyntheticBoolLiteral = 11
    BoolLiteral = 12
    Quote = 13
    SliceBegin = 14
    SliceEnd = 15
    SliceDelimiter = 16
    NakedSliceDelimiter = 17
    MarkerEnd = 18
    Warning = 19
    EOF = 20


class Position(NamedTuple):  # position.go:12-15
    line: int
    column: int


class Lexeme(NamedTuple):  # lexeme.go:32-36
    type: LexemeType
    value: bytes
    pos: Position


ZERO_LEXEME = Lexeme(LexemeType.Error, b"", Position(0, 0))


class Lexer:
    """One document's lexeme stream (NewLexer/Run/NextLexeme), replayed from GPU tuples."""

    def __init__(self, doc: bytes, tuples: np.ndarray):
        self._L = _native.lib()
        self._doc = bytes(doc)
        self._tuples = np.ascontiguousarray(tuples, dtype=np.uint64)
        self._h = self._L.obm_stream_new(self._doc, len(self._doc), self._tuples.ctypes.data, len(self._tuples))
        if not self._h:
            raise MemoryError("obm_stream_new")

    def run(self):
        """lexer.go:43 -- the scan already happened on the GPU; kept for interface parity."""

    def next_lexeme(self) -> Lexeme:
        lx = ObmLexeme()
        if not self._L.obm_stream_next(self._h, ctypes.byref(lx)):
            return ZERO_LEXEME
        return Lexeme(LexemeType(lx.type), ctypes.string_at(lx.value, lx.value_len), Position(lx.line, lx.column))

    def __iter__(self):
        while True:
            lx = self.next_lexeme()
            if lx is ZERO_LEXEME:
                return
            yield lx

    def close(self):
        if self._h:
            self._L.obm_stream_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def decode_doc_raw(doc: bytes, tuples: np.ndarray) -> bytes:
    """Whole-document decode into the flat record format [u8 type][u32 line][u32 col][u32 vlen][value]..."""
    L = _native.lib()
    tuples = np.ascontiguousarray(tuples, dtype=np.uint64)
    out = ctypes.POINTER(ctypes.c_uint8)()
    outlen = ctypes.c_uint64()
    n = L.obm_decode_doc(doc, len(doc), tuples.ctypes.data, len(tuples), ctypes.byref(out), ctypes.byref(outlen))
    if n < 0:
        raise NativeError(n, "obm_decode_doc")
    data = ctypes.string_at(out, outlen.value)
    L.obm_free(out)
    return data


class BatchResult(NamedTuple):
    tuples: np.ndarray         # uint64[n_tuples]
    doc_tuple_off: np.ndarray  # uint64[ndocs+1]
    stats: dict


class Scanner:
    """Owns one obm_handle (one GPU, one stream): the batch replacement for `NewLexer` per document."""

    def __init__(self, device: int = 0):
        self._L = _native.lib()
        h = ctypes.c_void_p()
        rc = self._L.obm_create(device, ctypes.byref(h))
        if rc != 0:
            raise NativeError(rc, self._L.obm_last_error(None).decode())
        self._h = h
        self.device = device

    @property
    def handle(self):
        return self._h

    def _check(self, rc):
        if rc != 0:
            raise NativeError(rc, self._L.obm_last_error(self._h).decode())

    def set_mode(self, mode: int) -> int:
        return self._L.obm_set_mode(self._h, mode)

    def set_chunk_bytes(self, nbytes: int) -> int:
        return self._L.obm_set_chunk_bytes(self._h, nbytes)

    def lex_batch(self, data, doc_off, out: np.ndarray = None) -> BatchResult:
        """data: bytes-like / uint8 array of packed documents; doc_off: uint64[ndocs+1]."""
        buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
        ndocs = len(doc_off) - 1
        toff = np.zeros(ndocs + 1, dtype=np.uint64)
        cnt = ctypes.c_uint64()
        st = ObmStats()
        if out is None:
            # size first (count pass only), then fill
            rc = self._L.obm_lex_batch(self._h, buf.ctypes.data, doc_off.ctypes.data, ndocs, None, 0, ctypes.byref(cnt),
                                       toff.ctypes.data, ctypes.byref(st))
            if rc not in (0, _native.OBM_E_CAPACITY):
                self._check(rc)
            out = np.empty(max(int(cnt.value), 1), dtype=np.uint64)
        rc = self._L.obm_lex_batch(self._h, buf.ctypes.data, doc_off.ctypes.data, ndocs, out.ctypes.data, len(out),
                                   ctypes.byref(cnt), toff.ctypes.data, ctypes.byref(st))
        self._check(rc)
        stats = {f: getattr(st, f) for f, _ in ObmStats._fields_}
        return BatchResult(out[:cnt.value], toff, stats)

    def parse_batch(self, registry: "Registry", data, doc_off, res_cap: int = None, arg_cap: int = None,
                    host_cap: int = None) -> "ParseBatchResult":
        """The parser over a host batch in one device call (include/obmarkers.h: obm_parse_batch): H2D, scan, parse, and
        back only the Result records plus the tuples of the documents the host must parse itself.  Without capacities a
        sizing call comes first; with them, too small a capacity raises NativeError (OBM_E_CAPACITY)."""
        buf = np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data
        doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
        ndocs = len(doc_off) - 1
        roff = np.zeros(ndocs + 1, dtype=np.uint64)
        hoff = np.zeros(ndocs + 1, dtype=np.uint64)
        totals = np.zeros(3, dtype=np.uint64)
        st = ObmStats()
        if res_cap is None or arg_cap is None or host_cap is None:
            rc = self._L.obm_parse_batch(self._h, registry.handle, buf.ctypes.data, doc_off.ctypes.data, ndocs, None, 0, None, 0,
                                         roff.ctypes.data, None, 0, hoff.ctypes.data, totals.ctypes.data, ctypes.byref(st))
            if rc not in (0, _native.OBM_E_CAPACITY):
                self._check(rc)
            res_cap, arg_cap, host_cap = (int(x) for x in totals)
        res = np.empty(max(res_cap, 1), dtype=RESULT_DT)
        args = np.empty(max(arg_cap, 1), dtype=ARG_DT)
        host = np.empty(max(host_cap, 1), dtype=np.uint64)
        rc = self._L.obm_parse_batch(self._h, registry.handle, buf.ctypes.data, doc_off.ctypes.data, ndocs, res.ctypes.data, res_cap,
                                     args.ctypes.data, arg_cap, roff.ctypes.data, host.ctypes.data, host_cap, hoff.ctypes.data,
                                     totals.ctypes.data, ctypes.byref(st))
        self._check(rc)
        stats = {f: getattr(st, f) for f, _ in ObmStats._fields_}
        nres, nargs, nhost = (int(x) for x in totals)
        return ParseBatchResult(registry, res[:nres], args[:nargs], roff, host[:nhost], hoff, stats)

    def lex_batch_device(self, d_bytes, d_doc_off, ndocs, total_bytes, d_out, out_cap, d_tuple_off, d_status=None,
                         d_counts=None, stream=None):
        """Raw device-pointer entry point (ints / torch .data_ptr()). Asynchronous."""
        self._check(self._L.obm_lex_batch_device(self._h, d_bytes, d_doc_off, ndocs, total_bytes, d_out, out_cap,
                                                 d_tuple_off, d_status, d_counts, stream))

    def lex_collection_batch_device(self, d_bytes, d_doc_off, ndocs, total_bytes, d_out_bytes, out_bytes_cap, d_out_doc_off, d_out, out_cap,
                                    d_tuple_off, d_status=None, d_counts=None, stream=None):
        """Manifest.LoadContent's rewrite of a collection batch, then lex_batch_device of the result (include/obmarkers.h:
        obm_lex_collection_batch_device): writes the rewritten bytes (d_out_bytes, 16-byte aligned, out_bytes_cap >=
        total_bytes) and their offsets, and the tuples of the rewritten documents. Synchronises the stream."""
        self._check(self._L.obm_lex_collection_batch_device(self._h, d_bytes, d_doc_off, ndocs, total_bytes, d_out_bytes, out_bytes_cap,
                                                            d_out_doc_off, d_out, out_cap, d_tuple_off, d_status, d_counts, stream))

    def parse_batch_device(self, registry, d_bytes, d_doc_off, ndocs, doc_base, d_tuples, d_tuple_off, d_results, res_cap, d_args, arg_cap,
                           d_doc_res_off, d_totals=None, stream=None):
        """The parser on the device (include/obmarkers.h: obm_parse_batch_device). Asynchronous."""
        self._check(self._L.obm_parse_batch_device(self._h, registry.handle, d_bytes, d_doc_off, ndocs, doc_base, d_tuples, d_tuple_off, d_results,
                                                   res_cap, d_args, arg_cap, d_doc_res_off, d_totals, stream))

    def generate_corpus_device(self, d_bytes, d_doc_off, ndocs, doc_bytes, first_doc=0, flavour=0, stream=None):
        self._check(self._L.obm_generate_corpus_device(self._h, d_bytes, d_doc_off, ndocs, doc_bytes, first_doc, flavour, stream))

    def lexers(self, data, doc_off, result: BatchResult):
        """One Lexer per document, in order."""
        mv = memoryview(data)
        for d in range(len(doc_off) - 1):
            doc = bytes(mv[int(doc_off[d]):int(doc_off[d + 1])])
            yield Lexer(doc, result.tuples[int(result.doc_tuple_off[d]):int(result.doc_tuple_off[d + 1])])

    def close(self):
        if self._h:
            self._L.obm_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Comm:
    """One rank of the multi-GPU path (obm_comm_*): file shards, one NCCL all-gather of the compact Result records."""

    def __init__(self, scanner: Scanner, unique_id: bytes, rank: int, nranks: int):
        self._L = _native.lib()
        self.scanner, self.rank, self.nranks = scanner, rank, nranks
        c = ctypes.c_void_p()
        idbuf = (ctypes.c_uint8 * 128).from_buffer_copy(unique_id)
        rc = self._L.obm_comm_create(scanner.handle, idbuf, rank, nranks, ctypes.byref(c))
        if rc != 0:
            raise NativeError(rc, self._L.obm_last_error(scanner.handle).decode())
        self._c = c

    @staticmethod
    def unique_id() -> bytes:
        L = _native.lib()
        buf = (ctypes.c_uint8 * 128)()
        rc = L.obm_comm_unique_id(buf)
        if rc != 0:
            raise NativeError(rc, L.obm_last_error(None).decode())
        return bytes(buf)

    def lex_batch_sharded_device(self, registry, d_bytes, d_doc_off, ndocs, total_bytes, first_doc, d_out, out_cap, d_tuple_off, d_status, d_counts,
                                 d_index, index_cap, d_index_all, index_all_cap, stream=None):
        """scan + marker index + one all-gather of the index records -> (records per rank, slot stride); the all-gather is
        enqueued on `stream`"""
        per_rank = (ctypes.c_uint64 * self.nranks)()
        stride = ctypes.c_uint64()
        rc = self._L.obm_lex_batch_sharded_device(self._c, registry.handle, d_bytes, d_doc_off, ndocs, total_bytes, first_doc, d_out, out_cap,
                                                  d_tuple_off, d_status, d_counts, d_index, index_cap, d_index_all, index_all_cap,
                                                  per_rank, ctypes.byref(stride), stream)
        if rc != 0:
            raise NativeError(rc, self._L.obm_last_error(self.scanner.handle).decode())
        return list(per_rank), int(stride.value)

    def close(self):
        if self._c:
            self._L.obm_comm_destroy(self._c)
            self._c = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def generate_corpus_host(ndocs: int, doc_bytes: int = 4096, first_doc: int = 0, flavour: int = 0):
    """Host copy of the device corpus generator -> (uint8[ndocs*doc_bytes], uint64[ndocs+1])."""
    L = _native.lib()
    data = np.empty(ndocs * doc_bytes, dtype=np.uint8)
    off = np.empty(ndocs + 1, dtype=np.uint64)
    rc = L.obm_generate_corpus_host(data.ctypes.data, off.ctypes.data, ndocs, doc_bytes, first_doc, flavour)
    if rc != 0:
        raise NativeError(rc, "obm_generate_corpus_host")
    return data, off


# ---- the lexer's consumer: internal/markers/parser over the same tuple stream (SURVEY.md 8(f) rank 1) ----
FIELD_MARKER, COLLECTION_MARKER, RESOURCE_MARKER = 0, 1, 2  # internal/workload/v1/markers/markers.go:20-25


class Registry:
    """marker.Registry stand-in (marker/registry.go:8-42): marker names (with '+') -> accepted argument names.

    Registry() and Registry({name: args}) hold names only: every argument value is accepted and every marker emits.
    Registry.define(FIELD_MARKER, ...) holds the typed definitions marker.Define builds from operator-builder's structs,
    so Results carry SetArgument / InflateObject's errors (include/obmarkers.h: obm_registry_define)."""

    @classmethod
    def define(cls, *marker_types):
        """A registry of the typed definitions of `marker_types` (FIELD_MARKER, COLLECTION_MARKER, RESOURCE_MARKER), like
        InspectForYAML(..., markerTypes...) builds (markers.go:92-113)."""
        r = cls({})
        for t in marker_types:
            r.define_marker(t)
        return r

    def define_marker(self, marker_type: int):
        """Add (or replace, by name) the typed definition of one marker type."""
        rc = self._L.obm_registry_define(self._r, int(marker_type))
        if rc != 0:
            raise NativeError(rc, f"obm_registry_define: unknown marker type {marker_type}")
        return self

    def __init__(self, markers=None):
        self._L = _native.lib()
        if markers is None:
            self._r = self._L.obm_registry_operator_builder()  # field / collection:field / resource
        else:
            self._r = self._L.obm_registry_new()
            for name, args in markers.items():
                arr = (ctypes.c_char_p * max(1, len(args)))(*[a if isinstance(a, bytes) else a.encode() for a in args])
                self._L.obm_registry_add(self._r, name if isinstance(name, bytes) else name.encode(), arr, len(args))

    @property
    def handle(self):
        return self._r

    def __del__(self):
        try:
            if self._r:
                self._L.obm_registry_free(self._r)
                self._r = None
        except Exception:
            pass


def parse_doc_raw(registry: Registry, doc: bytes, tuples: np.ndarray) -> bytes:
    """parser.NewParser(...).Parse() over one document's tuples -> serialised Results (csrc/obm_parse.cpp)."""
    L = _native.lib()
    tuples = np.ascontiguousarray(tuples, dtype=np.uint64)
    out = ctypes.POINTER(ctypes.c_uint8)()
    outlen = ctypes.c_uint64()
    n = L.obm_parse_doc(registry.handle, doc, len(doc), tuples.ctypes.data, len(tuples), ctypes.byref(out), ctypes.byref(outlen))
    if n < 0:
        raise NativeError(n, "obm_parse_doc")
    data = ctypes.string_at(out, outlen.value)
    L.obm_free(out)
    return data


# obm_result / obm_arg (include/obmarkers.h): the records k_parse_docs writes
RESULT_DT = np.dtype([("doc", "<u4"), ("tuple", "<u4"), ("text_off", "<u4"), ("text_len", "<u4"), ("reg_id", "<u2"), ("nargs", "<u2"),
                      ("arg_base", "<u4"), ("flags", "<u4"), ("aux", "<u4")])
ARG_DT = np.dtype([("name_off", "<u4"), ("val_off", "<u4"), ("val_len", "<u4"), ("name_len", "<u2"), ("kind", "u1"), ("flags", "u1")])
R_OK, R_NL, R_ERR_PARSEBOOL, R_ERR_FLOAT32, R_HOST, R_ERR_SETARG, R_ERR_MISSING, R_PANIC = 1, 2, 4, 8, 16, 32, 64, 128
A_SYNTHETIC_TRUE, A_SUPERSEDED = 1, 2


def results_format_doc(registry: Registry, doc: bytes, tuples: np.ndarray, results: np.ndarray, args: np.ndarray) -> bytes:
    """One document's records (results: its slice; args: the batch's whole array) -> the byte format of parse_doc_raw.
    A document whose record is R_HOST is parsed from `tuples` (obm_results_format_doc)."""
    L = _native.lib()
    tuples = np.ascontiguousarray(tuples, dtype=np.uint64)
    results = np.ascontiguousarray(results, dtype=RESULT_DT)
    args = np.ascontiguousarray(args, dtype=ARG_DT)
    out = ctypes.POINTER(ctypes.c_uint8)()
    outlen = ctypes.c_uint64()
    n = L.obm_results_format_doc(registry.handle, doc, len(doc), tuples.ctypes.data, len(tuples), results.ctypes.data, len(results),
                                 args.ctypes.data if len(args) else None, ctypes.byref(out), ctypes.byref(outlen))
    if n < 0:
        raise NativeError(n, "obm_results_format_doc")
    data = ctypes.string_at(out, outlen.value)
    L.obm_free(out)
    return data


class ParseBatchResult(NamedTuple):
    """What Scanner.parse_batch returns: document d's Results are results[doc_res_off[d]:doc_res_off[d+1]] (their arg_base
    indexes `args` as a whole); its tuples are host_tuples[doc_host_off[d]:doc_host_off[d+1]], present only when its one
    record is R_HOST."""
    registry: Registry
    results: np.ndarray       # RESULT_DT[n_results]
    args: np.ndarray          # ARG_DT[n_args]
    doc_res_off: np.ndarray   # uint64[ndocs+1]
    host_tuples: np.ndarray   # uint64[n_fallback_tuples]
    doc_host_off: np.ndarray  # uint64[ndocs+1]
    stats: dict

    def format_doc(self, d: int, doc: bytes) -> bytes:
        """document d's Results in parse_doc_raw's byte format (doc: its bytes)"""
        r = self.results[int(self.doc_res_off[d]):int(self.doc_res_off[d + 1])]
        t = self.host_tuples[int(self.doc_host_off[d]):int(self.doc_host_off[d + 1])]
        return results_format_doc(self.registry, doc, t, r, self.args)
