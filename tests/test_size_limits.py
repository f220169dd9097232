"""The tuple format at its size limits (include/obmarkers.h): slices longer than OBM_MAX_LEN = 2^27 - 1 go out as PART
pieces, line numbers above 2^27 are announced by LINEHI, documents may be up to OBM_MAX_DOC_BYTES = 2^31 - 2 bytes.

One case list serves every layer:
- on the CPU, the exact lexer, its line-mode composition and the replay of the chunk-parallel large path
  (hostsim.large_doc) must all decode to what the oracle gives, and every PART piece but the last of a chain is
  exactly OBM_MAX_LEN long; the host consumers (the Lexer stream replay, parse_doc_raw) read such streams;
- on the GPU, every mode must give the host exact lexer's tuples bit for bit (which the CPU tests tie to the oracle),
  between small documents in one shot and alone chunked (modes 0, 2, 3 on GPU_CASES, mode 1 on EXACT_MODE_CASES); the
  hash leaves these documents to the host; parse_batch hands them back as OBM_R_HOST; the flat marker index finds a
  marker after 2^27 lines;
- one document of exactly 2^31 - 2 bytes goes through lex_batch_device's large path (modes 0, 2, 3).

Documents are 128-256 MiB each, so they are built one at a time and tuple arrays are sized by a counting pass.
"""
import ctypes
import hashlib
import random
import time

import numpy as np
import pytest

from tests import hostsim

LEN_BITS = 27
MAX_LEN = (1 << LEN_BITS) - 1            # OBM_MAX_LEN
MAX_DOC = (1 << 31) - 2                  # OBM_MAX_DOC_BYTES
LONG = (1 << LEN_BITS) + 1
K_PART, K_DRIFT, K_LINEHI, K_ERR_FLOAT, K_ERR_INT = 21, 23, 25, 30, 31
LEX_ERROR = 0

ASCII_LEAD, UNI_LEAD = b"# e\n", "# é\n".encode()   # a comment line before the case; the second makes it non-ASCII


def _long_bodies():
    """(name, body): every lexeme kind that can carry a slice longer than OBM_MAX_LEN"""
    out = [(f"dq{n - LONG:+d}", b'# +a:b="' + b"x" * n + b'",c\n# tail\n') for n in (LONG - 2, LONG - 1, LONG)]
    out += [("dq-two-pieces", b'# +a:b="' + b"x" * (2 * (1 << LEN_BITS) + 3) + b'",c\n'),
            ("backtick", b"# +a:b=`" + b"x" * LONG + b"`,c\n# +d:e=1\n"),
            ("backtick-lines", b"# +a:b=`" + b"x" * LONG + b"\n  # w`\n# tail\n"),   # multi-line: the sequential fallback
            ("arg-name", b"# +a:b=1," + b"y" * LONG + b"=2\n"),
            ("scope-warning", b"# +" + b"s" * LONG + b"\n# +c:d=1\n"),              # WARN_NOSCOPE after a stale buffer
            ("int-overflow", b"# +a:b=" + b"1" * LONG + b"\n"),
            ("float-overflow", b"# +a:b=" + b"9" * LONG + b".5\n"),
            ("float-long-ok", b"# +a:b=1." + b"0" * LONG + b",c\n")]
    return out


# a marker line, one whose drift (a backed-up rune, state.go:79) shifts a warning's column, and one warning
LINE_TAIL = b"# +a:b=1,c\n# +a:,+b c\n+q\n"
LINE_COUNTS = ((1 << LEN_BITS) - 1, 1 << LEN_BITS, (1 << LEN_BITS) + 1, (1 << (LEN_BITS + 1)) + 5)

CASES = [f"{name}/{lead}" for name, _b in _long_bodies() for lead in ("ascii", "uni")]
CASES += [f"lines{k}/ascii" for k in LINE_COUNTS] + [f"lines{1 << LEN_BITS}/uni"]
# On the GPU, modes 0, 2 and 3: the cases the chunk-parallel large path lexes (both of its lexers, slices of exactly
# 2^27 - 1 bytes, one and two full PART pieces, a long name).  A case with a fatal error or a literal across lines falls
# back to one thread per document there, as mode 1 always does: minutes per case for what the CPU tests already check on
# the same source, so mode 1 takes one case of each of those families.
GPU_CASES = ["dq-2/ascii", "dq-2/uni", "dq-1/ascii", "dq+0/ascii", "dq-two-pieces/ascii", "backtick/ascii", "arg-name/ascii"]
EXACT_MODE_CASES = ["scope-warning/uni", "int-overflow/ascii", f"lines{(1 << LEN_BITS) + 1}/ascii"]


def case_doc(case: str) -> bytes:
    name, lead = case.split("/")
    pre = UNI_LEAD if lead == "uni" else ASCII_LEAD
    if name.startswith("lines"):
        # the tail's first line is line k (the lead is one of the k - 1 lines before it)
        return pre + b"\n" * (int(name[5:]) - 2) + LINE_TAIL
    return pre + dict(_long_bodies())[name]


def count_then_lex(fn, doc: bytes):
    """fn(doc, n, out, cap) -> tuple count: one counting call (cap 0), then exactly the room the stream needs"""
    n = fn(doc, len(doc), None, 0)
    out = np.zeros(max(1, n), dtype=np.uint64)
    assert fn(doc, len(doc), out.ctypes.data, n) == n
    return out[:n]


def exact_tuples(doc: bytes):
    L = hostsim.lib()
    return count_then_lex(lambda d, n, o, c: L.hs_lex_doc(d, n, o, c, None, None), doc)


def line_mode_tuples(doc: bytes):
    return count_then_lex(hostsim.lib().hs_lex_doc_by_lines, doc)


def large_path_tuples(doc: bytes):
    L = hostsim.lib()
    used = ctypes.c_uint32(0)
    t = count_then_lex(lambda d, n, o, c: L.hs_large_doc(d, n, o, c, ctypes.byref(used)), doc)
    return t, bool(used.value)


def kinds(t):
    return (np.asarray(t, dtype=np.uint64) >> np.uint64(59)).astype(np.int64)


def lens(t):
    return ((np.asarray(t, dtype=np.uint64) >> np.uint64(32)) & np.uint64(MAX_LEN)).astype(np.int64)


def offs(t):
    return (np.asarray(t, dtype=np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.int64)


def check_part_chains(t):
    """every PART that continues into the next tuple's slice is a full piece of OBM_MAX_LEN bytes (a PART of the stale
    buffer before a warning or a FLUSH may be shorter: the pending text, not a split)"""
    k, ln, of = kinds(t), lens(t), offs(t)
    for i in np.nonzero(k == K_PART)[0]:
        if i + 1 < len(t) and (k[i + 1] == K_PART or 1 <= k[i + 1] <= 13 or k[i + 1] in (K_ERR_FLOAT, K_ERR_INT)) \
                and of[i + 1] == of[i] + ln[i]:
            assert ln[i] == MAX_LEN, (i, hostsim.fmt_tuples(t[max(0, i - 2):i + 3]))


def decoded_digest(doc, t):
    return hashlib.sha256(hostsim.decode(doc, t)).hexdigest()


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the host build of the lexers against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_lexers_match_oracle(oracle, case):
    doc = case_doc(case)
    want = hashlib.sha256(oracle.lex_raw(doc)).hexdigest()
    exact = exact_tuples(doc)
    assert decoded_digest(doc, exact) == want, ("exact", case, hostsim.fmt_tuples(exact)[:24])
    check_part_chains(exact)
    k = kinds(exact)
    if case.startswith("lines"):
        assert (k == K_LINEHI).any() and (k == K_DRIFT).any(), case
    else:
        assert (k == K_PART).any() == (not case.startswith("dq-2/")), case   # 2^27 - 1 bytes still fit one tuple
    assert np.array_equal(line_mode_tuples(doc), exact), case
    large, chained = large_path_tuples(doc)
    fatal = (k == K_ERR_FLOAT).any() or (k == K_ERR_INT).any()
    assert chained == (not case.startswith("backtick-lines") and not fatal), case   # otherwise: the sequential fallback
    assert np.array_equal(large, exact), ("large path", case, hostsim.fmt_tuples(large)[:24], hostsim.fmt_tuples(exact)[:24])


def test_numeric_errors_quote_the_whole_literal(oracle):
    """the oracle's message quotes the whole literal, with its end as the column: ERR_INT / ERR_FLOAT keep off + len at the
    literal's end, after PART pieces of OBM_MAX_LEN"""
    for body, kind in ((b"# +a:b=" + b"1" * LONG + b"\n", K_ERR_INT), (b"# +a:b=" + b"9" * LONG + b".5\n", K_ERR_FLOAT)):
        t = exact_tuples(body)
        k, ln, of = kinds(t), lens(t), offs(t)
        e = int(np.nonzero((k == K_ERR_INT) | (k == K_ERR_FLOAT))[0][0])
        assert k[e] == kind and k[e - 1] == K_PART and ln[e - 1] == MAX_LEN and of[e] + ln[e] == len(body) - 1
        err = [val for typ, val, _l, _c in oracle.parse_stream(hostsim.decode(body, t)) if typ == LEX_ERROR]
        assert len(err) == 1 and b"value out of range" in err[0] and err[0].count(body[7:-1]) == 2, err[0][-80:]


def chunk_starts_reference(doc: bytes):
    """first line start at or after c * 1024 (n if none) and 1 + the newlines before it, for every chunk"""
    n = len(doc)
    nl = np.nonzero(np.frombuffer(doc, np.uint8) == 10)[0]
    starts = np.concatenate([[0], nl + 1])
    nc = max(1, -(-n // 1024))
    idx = np.searchsorted(starts, np.arange(nc, dtype=np.int64) * 1024)
    cs = np.where(idx < len(starts), starts[np.minimum(idx, len(starts) - 1)], n)
    return cs.astype(np.uint32), (1 + np.searchsorted(nl, cs)).astype(np.uint32)


@pytest.mark.parametrize("seed", range(4))
def test_chunk_starts(seed):
    """resolved chunk starts of the large path (chunk_start + resolve_chunk_starts) on lines of 1 B to 40 KiB"""
    rng = random.Random(seed)
    parts, n = [], 0
    while n < (3 << 20):
        ln = rng.choice([0, 1, 2, rng.randrange(1, 1024), rng.randrange(1000, 1050), rng.randrange(1, 40 << 10)])
        parts.append(b"x" * ln + b"\n")
        n += ln + 1
    for doc in (b"".join(parts), b"".join(parts)[:-1], b"".join(parts)[rng.randrange(1, 4096):]):
        cs, line = hostsim.large_chunk_starts(doc)
        want_cs, want_line = chunk_starts_reference(doc)
        assert np.array_equal(cs, want_cs) and np.array_equal(line, want_line), seed


def test_chunk_starts_of_one_long_line_are_linear():
    """one 128 MiB line: every chunk looks at its own 1 KiB only (a search that runs on to the line's end reads about
    L^2 / 2048 bytes: hours on the CPU for this line)"""
    doc = b"# +a:b=" + b"v" * (1 << 27) + b"\nk: v # +c:d=1\n"
    t0 = time.perf_counter()
    cs, line = hostsim.large_chunk_starts(doc)
    assert time.perf_counter() - t0 < 30
    assert (cs[1:-1] == len(doc) - 14).all() and (line[1:-1] == 2).all()
    assert cs[0] == 0 and line[0] == 1


def test_stream_replay_past_the_limits(oracle):
    """the Lexer stream replay (obm_stream_next) over LINEHI lines and PART chains"""
    import operator_builder_b200 as ob
    doc = b"\n" * ((1 << LEN_BITS) + 4) + b'# +a:b="' + b"x" * LONG + b'",c\n'
    lx = list(ob.Lexer(doc, exact_tuples(doc)))
    s = [x for x in lx if x.type == ob.LexemeType.StringLiteral]
    assert len(s) == 1 and len(s[0].value) == LONG and s[0].value == b"x" * LONG
    assert s[0].pos.line == (1 << LEN_BITS) + 5 and s[0].pos.column == 9
    assert [int(x.type) for x in lx] == [typ for typ, _v, _l, _c in oracle.lex(doc)]


def test_parse_doc_raw_past_the_limits(oracle):
    """parse_doc_raw equals the parser oracle for a registered marker with a 128 MiB value and after 2^27 lines"""
    import operator_builder_b200 as ob
    from oracle import parser_oracle as po
    reg = ob.Registry()
    for doc in (b'# +operator-builder:field:name=x,default="' + b"d" * LONG + b'",type=string\n',
                b"\n" * ((1 << LEN_BITS) + 1) + b"# +operator-builder:field:name=x,type=int\n"):
        want = po.serialize(po.parse(oracle.lex(doc), po.OPERATOR_BUILDER_REGISTRY))
        assert ob.parse_doc_raw(reg, doc, exact_tuples(doc)) == want
        assert b"operator-builder:field" in want


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
SMALL = [b"k: v # +s:a=1\n", b"", b"# +x:y=\"q\"\n", "# é +a:b=ü\n".encode(), b"+a:b=1e309\n"]


def pack(docs):
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    data = np.empty(int(off[-1]), dtype=np.uint8)
    for d, o in zip(docs, off):
        data[int(o):int(o) + len(d)] = np.frombuffer(d, np.uint8)
    return data, off


@pytest.fixture(scope="module")
def scanner():
    import operator_builder_b200 as ob
    sc = ob.Scanner(0)
    yield sc
    sc.set_mode(0)
    sc.close()


def device_hash_check(scanner, oracle, docs, data, off, res, want):
    """obm_hash_batch_device: the documents with a PART, LINEHI or other pseudo-tuple get hash 0 and are counted in n_host,
    the others get FNV-1a of their decoded stream"""
    import torch
    import operator_builder_b200 as ob
    from operator_builder_b200 import _native
    from tests import test_stream_consumers as tsc
    n = len(docs)
    d_bytes, d_off, d_tup, d_toff = tsc.to_dev(data), tsc.to_dev(off), tsc.to_dev(res.tuples), tsc.to_dev(res.doc_tuple_off)
    d_hash = torch.full((n,), 0x1234, dtype=torch.int64, device="cuda:0")
    d_nh = torch.full((1,), 77, dtype=torch.int32, device="cuda:0")
    assert _native.lib().obm_hash_batch_device(scanner.handle, d_bytes.data_ptr(), d_off.data_ptr(), n, d_tup.data_ptr(), d_toff.data_ptr(),
                                               d_hash.data_ptr(), d_nh.data_ptr(), tsc._stream()) == 0
    torch.cuda.synchronize()
    got = d_hash.cpu().numpy().view(np.uint64)
    flagged = [tsc.host_flag(d, w) for d, w in zip(docs, want)]
    for i, d in enumerate(docs):
        if flagged[i]:
            assert int(got[i]) == 0, i
        elif len(d) < (1 << 20):
            assert int(got[i]) == tsc.fnv1a(ob.decode_doc_raw(d, want[i])), i
        else:   # FNV-1a of a 128 MiB stream in Python takes minutes: the oracle's own per-document hash
            one, one_off = pack([d])
            assert int(got[i]) == int(oracle.scan_batch(one, one_off, 4, want_doc_hash=True)[3][0]) != 0, i
    assert int(d_nh.item()) == sum(flagged)


def device_lex_check(scanner, case, modes):
    """lex_batch in one shot between small documents and chunked alone: the host exact lexer's tuples bit for bit"""
    doc = case_doc(case)
    want = exact_tuples(doc)
    docs = SMALL[:3] + [doc] + SMALL[3:]
    small_want = [exact_tuples(d) for d in docs]
    expect = np.concatenate(small_want)
    data, off = pack(docs)
    data1, off1 = pack([doc])
    try:
        for mode in modes:
            scanner.set_mode(mode)
            res = scanner.lex_batch(data, off, out=np.empty(len(expect), np.uint64))
            assert np.array_equal(res.tuples, expect), (case, mode)
            assert np.array_equal(np.diff(res.doc_tuple_off.astype(np.int64)), [len(w) for w in small_want]), (case, mode)
            old = scanner.set_chunk_bytes(1 << 20)
            try:
                res1 = scanner.lex_batch(data1, off1, out=np.empty(len(want), np.uint64))
            finally:
                scanner.set_chunk_bytes(old)
            assert np.array_equal(res1.tuples, want), (case, mode, "chunked")
    finally:
        scanner.set_mode(0)
    return doc, want, docs, small_want, data, off, res


@pytest.mark.gpu
@pytest.mark.parametrize("case", EXACT_MODE_CASES)
def test_device_exact_mode(scanner, case):
    """mode 1 (the exact path, one thread per document) gives the same tuples as the large path"""
    device_lex_check(scanner, case, (1,))


@pytest.mark.gpu
@pytest.mark.parametrize("case", GPU_CASES)
def test_device_modes(scanner, oracle, case):
    """modes 0, 2 and 3 (the chunk-parallel large path) give the host exact lexer's tuples bit for bit.  The hash leaves
    a document with PART or LINEHI tuples to the host and hashes the others right; parse_batch hands the former back
    as one OBM_R_HOST record with its tuples"""
    import operator_builder_b200 as ob
    doc, want, docs, small_want, data, off, res = device_lex_check(scanner, case, (0, 2, 3))
    device_hash_check(scanner, oracle, docs, data, off, res, small_want)
    reg = ob.Registry()
    parsed = scanner.parse_batch(reg, data, off)
    if not case.startswith("dq-2/"):
        r = parsed.results[int(parsed.doc_res_off[3]):int(parsed.doc_res_off[4])]
        assert len(r) == 1 and int(r[0]["flags"]) & ob.lexer.R_HOST
        assert np.array_equal(parsed.host_tuples[int(parsed.doc_host_off[3]):int(parsed.doc_host_off[4])], want)
    for i, d in enumerate(docs):
        assert parsed.format_doc(i, d) == ob.parse_doc_raw(reg, d, small_want[i]), (case, i)


@pytest.mark.gpu
def test_device_parse_batch_registered_markers(scanner, oracle):
    """parse_batch's gathered tuples of a registered marker with a 128 MiB value and one after 2^27 lines give
    parse_doc_raw's Results and the parser oracle's"""
    import operator_builder_b200 as ob
    from oracle import parser_oracle as po
    docs = [b'# +operator-builder:field:name=x,default="' + b"d" * LONG + b'",type=string\n', SMALL[0],
            b"\n" * ((1 << LEN_BITS) + 1) + b"# +operator-builder:field:name=x,type=int\n"]
    reg = ob.Registry()
    data, off = pack(docs)
    parsed = scanner.parse_batch(reg, data, off)
    for i, d in enumerate(docs):
        want = po.serialize(po.parse(oracle.lex(d), po.OPERATOR_BUILDER_REGISTRY))
        assert parsed.format_doc(i, d) == ob.parse_doc_raw(reg, d, exact_tuples(d)) == want, i


@pytest.mark.gpu
def test_device_flat_index_after_2p27_lines(scanner, oracle):
    """obm_marker_index_flat_device: a registered marker on line 2^27 + 2 agrees with obm_marker_index_device and the
    parser oracle's loaded definitions"""
    from tests import test_stream_consumers as tsc
    doc = b"\n" * ((1 << LEN_BITS) + 1) + b"# +operator-builder:field:name=x\n" + b"k: v # +operator-builder:resource:field=a\n"
    tsc.check_flat(scanner, oracle, tsc.OB, [SMALL[0], doc, tsc.MARKER], min_records=3)


def shifted(stream: bytes, lines: int) -> bytes:
    """a serialised lexeme stream with every located Pos.line moved down by `lines` (synthetic lexemes have line 0)"""
    import oracle as o
    out = bytearray()
    for typ, val, line, col in o.parse_stream(stream):
        out += bytes([typ]) + np.array([line + lines if line else 0, col, len(val)], "<u4").tobytes() + val
    return bytes(out)


def big_doc_tail(seed=7, size=4096):
    """markers, comments and plain lines, no warnings and no errors (their messages print positions as text)"""
    rng = random.Random(seed)
    pool = [b"# +operator-builder:field:name=a.b,type=int,default=3\n", b"k: v  # +s:a=1,b\n", b"# plain\n", b"\n",
            b"x: 'q'  # +x:y=\"s t\",z\n", b"- item # +a:b=`c`\n", b"path: /a/b\n"]
    parts, n = [], 0
    while n < size:
        ln = rng.choice(pool)
        parts.append(ln)
        n += len(ln)
    return b"".join(parts)


def big_doc_prefix(n_bytes: int) -> bytes:
    """`k: v` lines (no tuples) filling exactly n_bytes (a multiple of 5 or at least 9), ending in a newline"""
    r = n_bytes % 5
    head = b"k: v" + b"v" * (5 + r) + b"\n" if r else b""
    return head + b"k: v\n" * ((n_bytes - len(head)) // 5)


@pytest.mark.parametrize("prefix", [1 << 20, 1 << 27])
def test_shifted_tail_reference(oracle, prefix):
    """the 2 GiB test's reference: the oracle on the tail alone, lines shifted, equals the oracle on prefix + tail"""
    tail = big_doc_tail()
    pre = big_doc_prefix(prefix + 3)
    assert len(pre) == prefix + 3
    assert shifted(oracle.lex_raw(tail), pre.count(b"\n")) == oracle.lex_raw(pre + tail)


@pytest.mark.gpu
def test_device_2gib_document(scanner, oracle):
    """one document of exactly OBM_MAX_DOC_BYTES between small documents through lex_batch_device's large path (modes 0,
    2 and 3; mode 1 would lex the 2 GiB on one GPU thread and is left out): the tail's offsets reach past 2^31 - 4 KiB and
    its lines need LINEHI"""
    import torch
    import operator_builder_b200 as ob
    from tests import test_stream_consumers as tsc
    tail = big_doc_tail()
    pre = big_doc_prefix(MAX_DOC - len(tail))
    lines = pre.count(b"\n")
    assert lines >= (1 << LEN_BITS)
    doc = pre + tail
    del pre
    assert len(doc) == MAX_DOC
    docs = SMALL[:2] + [doc] + SMALL[2:]
    data, off = pack(docs)
    want_small = [exact_tuples(d) for d in SMALL]
    want_doc = shifted(oracle.lex_raw(tail), lines)
    d_bytes, d_off = tsc.to_dev(data), tsc.to_dev(off)
    cap = 1 << 16
    for mode in (0, 2, 3):
        scanner.set_mode(mode)
        d_out = torch.full((cap,), -1, dtype=torch.int64, device="cuda:0")
        d_toff = torch.zeros(len(docs) + 1, dtype=torch.int64, device="cuda:0")
        d_status = torch.zeros(4, dtype=torch.int32, device="cuda:0")
        scanner.lex_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), len(docs), len(data), d_out.data_ptr(), cap,
                                 d_toff.data_ptr(), d_status.data_ptr(), None, tsc._stream())
        torch.cuda.synchronize()
        assert d_status.cpu().tolist()[0] == 0, mode
        toff = d_toff.cpu().numpy().view(np.uint64)
        tup = d_out.cpu().numpy().view(np.uint64)[:int(toff[-1])]
        got = [tup[int(toff[i]):int(toff[i + 1])] for i in range(len(docs))]
        assert (kinds(got[2]) == K_LINEHI).any() and offs(got[2]).max() > MAX_DOC - 4096, mode
        assert ob.decode_doc_raw(doc, got[2]) == want_doc, mode
        for g, w in zip(got[:2] + got[3:], want_small):
            assert np.array_equal(g, w), mode
    scanner.set_mode(0)


@pytest.mark.gpu
def test_lex_batch_refuses_a_document_over_the_limit(scanner):
    """a document of 2^31 - 1 bytes, backed by a real host buffer: OBM_E_ARG"""
    import operator_builder_b200 as ob
    from operator_builder_b200 import _native
    data = np.zeros(MAX_DOC + 1 + 8, dtype=np.uint8)
    for lens_ in ([MAX_DOC + 1], [4, MAX_DOC + 1, 3]):
        off = np.zeros(len(lens_) + 1, dtype=np.uint64)
        off[1:] = np.cumsum(lens_)
        with pytest.raises(ob.NativeError, match=f"error {_native.OBM_E_ARG}:"):
            scanner.lex_batch(data[:int(off[-1])], off, out=np.empty(16, np.uint64))
    off = np.array([0, MAX_DOC], dtype=np.uint64)          # the limit itself is accepted (sizing call only)
    cnt = ctypes.c_uint64()
    toff = np.zeros(2, dtype=np.uint64)
    rc = _native.lib().obm_lex_batch(scanner.handle, data.ctypes.data, off.ctypes.data, 1, None, 0, ctypes.byref(cnt), toff.ctypes.data, None)
    assert rc in (0, _native.OBM_E_CAPACITY)
