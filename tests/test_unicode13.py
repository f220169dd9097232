"""Unicode classes and %q quoting pinned to Go 1.16 (Unicode 13.0), on the host and through every GPU scan mode.

The reference lexer asks Go 1.16's unicode.IsLetter (after '+'), IsNumber (a numeric literal) and IsSpace (around
comments and bool literals), and quotes its own and the parser's messages with strconv.Quote, which escapes whatever
strconv.IsPrint rejects.  tests/golden/unicode13.json (tools/extract_unicode13.py: perl's `Present_In=13.0` and the
General_Category, checked against the published Unicode totals) is the one source those four classes are checked
against here, independently of the oracle, which shares the product's generated tables:

  - the fixture itself, and both generated headers (host GO_* and device D_GO_* arrays) against it;
  - every value from -1 to 0x110000 through the product's host classes (hostsim) and the oracle's;
  - strconv.Quote restated from Go 1.16's quote.go against the oracle's and the product's quoter, over every scalar value
    and the invalid UTF-8 shapes;
  - the sweep: every scalar value in five one-line contexts (+ the two-byte and invalid patterns in three), lexed by the
    product's host core + decoder and by the oracle, byte for byte; and what the lexer must do with each X -- a
    MarkerStart after '+' iff X is a letter, a number iff X is a number, '.' or '-', a BoolLiteral after X iff X is
    white space -- asserted from the fixture, so that a table regression fails even if oracle and product drift together;
  - parser messages (ParseBool, FieldType unmarshal) through obm_parse_doc against the parser oracles.
On the GPU the same sweep runs through obm_lex_batch in modes 0-3, obm_lex_batch_device at an odd address,
obm_hash_batch_device and obm_parse_batch."""
import functools
import json
import os
import random
import re

import numpy as np
import pytest

from tests import hostsim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NCP = 0x110000
CLASSES = ("letter", "number", "space", "print")  # bit k of obo_classify / hs_classify
CONTEXTS = {"marker": (b"+", b":a=1"), "name": (b"+a", b""), "value": (b"+a:b=", b""), "number": (b"+a:b=1", b""),
            "bool": (b"+a:b=", b"true")}
# invalid UTF-8: truncated 2/3/4-byte sequences, surrogates, overlongs, above U+10FFFF (lone bytes are added below)
INVALID = [b"\xc3", b"\xe2\x82", b"\xe2", b"\xf0\x9f\x98", b"\xf0\x9f", b"\xf0", b"\xed\xa0\x80", b"\xed\xbf\xbf",
           b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xf0\x80\x80\x80", b"\xf0\x8f\xbf\xbf",
           b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xf7\xbf\xbf\xbf", b"\xff\xfe"]
LONE = [bytes([b]) for b in range(0x80, 0x100)]


@functools.lru_cache(maxsize=None)
def fixture():
    with open(os.path.join(ROOT, "tests", "golden", "unicode13.json")) as f:
        return json.load(f)


@functools.lru_cache(maxsize=None)
def member(name):
    """bool[0x110000]: the fixture's class `name`"""
    m = np.zeros(NCP, dtype=bool)
    for lo, hi in fixture()[name]:
        m[lo:hi + 1] = True
    return m


def scalars():
    return np.r_[0:0xD800, 0xE000:NCP]


def cp_list(cps, limit=8):
    return ", ".join(f"U+{int(c):04X}" for c in cps[:limit]) + (f" ... ({len(cps)} in all)" if len(cps) > limit else "")


# ---------------------------------------------------------------------------------------------------------------------
# 1. the fixture, and the generated headers against it
# ---------------------------------------------------------------------------------------------------------------------
def test_fixture_counts_and_shape():
    u = fixture()
    want = {"letter": 131241, "number": 1781, "print": 143680, "space": 25}
    assert u["counts"] == want
    for name, n in want.items():
        rs = u[name]
        assert sum(hi - lo + 1 for lo, hi in rs) == n, name
        for (lo, hi), (lo2, _hi2) in zip(rs, rs[1:]):
            assert lo <= hi and hi + 1 < lo2, (name, lo, hi, lo2)  # sorted, disjoint, maximal
        assert 0 <= rs[0][0] and rs[-1][1] <= 0x10FFFF, name
        assert not any(lo <= 0xDFFF and hi >= 0xD800 for lo, hi in rs), name  # no surrogates
    assert not member("letter")[[0x08C8, 0x0C5D, 0x0CDD, 0x1B4C, 0x2C2F, 0xA7C0]].any()  # letters of Unicode 14.0 / 15.0
    assert not member("print")[[0x061D, 0x08C8, 0x0C3C, 0x0CF3, 0x0ECE, 0x180F]].any()
    # Go's Latin-1 rule and the White_Space code points above it
    assert np.flatnonzero(member("space")).tolist() == [9, 10, 11, 12, 13, 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B),
                                                        0x2028, 0x2029, 0x202F, 0x205F, 0x3000]
    assert member("letter")[[ord("a"), ord("Z"), 0xAA, 0xB5, 0xBA, 0x4E00]].all() and not member("letter")[[0x5F, 0xD7]].any()
    assert member("number")[[ord("0"), 0xB2, 0xBC, 0x0660, 0x2160]].all()
    assert member("print")[0x20] and not member("print")[[0x7F, 0xA0, 0xAD, 0x3000, 0x200B]].any()


def header_arrays(path):
    """{array name: [[lo, hi], ...]} of a generated header, parsed from its text"""
    with open(os.path.join(ROOT, path)) as f:
        text = f.read()
    out = {}
    for m in re.finditer(r"unsigned int (\w+)\[\]\[2\] = \{(.*?)\};", text, re.S):
        out[m.group(1)] = [[int(a, 16), int(b, 16)] for a, b in re.findall(r"\{0x([0-9A-F]+),0x([0-9A-F]+)\}", m.group(2))]
        assert f"#define {m.group(1)}_N {len(out[m.group(1)])}\n" in text, m.group(1)
    return out


@pytest.mark.parametrize("path", ["oracle/go_unicode_tables.h", "operator-builder_b200/csrc/go_unicode_tables.h"])
def test_headers_equal_fixture(path):
    u = fixture()
    arrays = header_arrays(path)
    want = {"GO_LETTER_RANGES": u["letter"], "GO_NUMBER_RANGES": u["number"], "GO_PRINT_RANGES": u["print"],
            "GO_SPACE_RANGES": u["space"]}
    if path.startswith("operator-builder_b200"):  # the device copies the exact path searches
        want.update(D_GO_LETTER_RANGES=u["letter"], D_GO_NUMBER_RANGES=u["number"])
    assert sorted(arrays) == sorted(want)
    for name, rs in want.items():
        assert arrays[name] == rs, name


# ---------------------------------------------------------------------------------------------------------------------
# 2. classification of every value
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("who", ["hostsim", "oracle"])
def test_classify_every_value(who, oracle):
    cps = np.arange(-1, NCP + 1, dtype=np.int32)
    got = hostsim.classify(cps) if who == "hostsim" else oracle.classify(cps)
    errors = []
    for k, name in enumerate(CLASSES):
        want = np.zeros(len(cps), dtype=bool)
        want[1:-1] = member(name)
        bad = cps[((got >> k) & 1).astype(bool) != want]
        if len(bad):
            errors.append(f"{name}: {len(bad)} code points differ from Unicode 13.0: {cp_list(bad)}")
    assert not errors, f"{who}: " + "; ".join(errors)


# ---------------------------------------------------------------------------------------------------------------------
# 3. strconv.Quote
# ---------------------------------------------------------------------------------------------------------------------
HEX = "0123456789abcdef"
ESCAPES = {0x07: "\\a", 0x08: "\\b", 0x0C: "\\f", 0x0A: "\\n", 0x0D: "\\r", 0x09: "\\t", 0x0B: "\\v"}


def decode_rune(s: bytes, i: int):
    """utf8.DecodeRune(s[i:]) -> (rune, width); (None, 1) for an invalid or short encoding"""
    c0 = s[i]
    if c0 < 0x80:
        return c0, 1
    k = 2 if 0xC2 <= c0 <= 0xDF else 3 if 0xE0 <= c0 <= 0xEF else 4 if 0xF0 <= c0 <= 0xF4 else 0
    try:  # Python's strict decoder rejects what DecodeRune rejects: overlongs, surrogates, > U+10FFFF, short input
        return (ord(s[i:i + k].decode("utf-8")), k) if k and i + k <= len(s) else (None, 1)
    except UnicodeDecodeError:
        return None, 1


def go_quote_ref(s: bytes) -> bytes:
    """strconv.Quote of Go 1.16 (quote.go appendQuotedWith / appendEscapedRune, quote '"', neither ASCII-only nor graphic),
    with IsPrint from the fixture"""
    printable = member("print")
    out, i = ['"'], 0
    while i < len(s):
        r, w = decode_rune(s, i)
        if r is None:
            out.append("\\x" + HEX[s[i] >> 4] + HEX[s[i] & 15])
        elif r in (0x22, 0x5C):
            out.append("\\" + chr(r))
        elif printable[r]:
            out.append(chr(r))
        elif r in ESCAPES:
            out.append(ESCAPES[r])
        elif r < 0x20:
            out.append(f"\\x{r:02x}")
        elif r < 0x10000:
            out.append(f"\\u{r:04x}")  # DEL included: Go 1.16 has no \x7f case
        else:
            out.append(f"\\U{r:08x}")
        i += w
    out.append('"')
    return "".join(out).encode("utf-8")


def test_quote_reference_spot_checks():
    """the restatement itself, on what Go 1.16 prints for these strings"""
    cases = {b"": b'""', b"a\"b\\": b'"a\\"b\\\\"', b"\x00\x07\x1b\x7f": b'"\\x00\\a\\x1b\\u007f"',
             "\u00a0\u3000\u200b\U000e0001".encode(): b'"\\u00a0\\u3000\\u200b\\U000e0001"',
             "\u00e9\u4e16\U0001f600".encode(): "\"\u00e9\u4e16\U0001f600\"".encode(),
             b"\xed\xa0\x80\xc0\x80": b'"\\xed\\xa0\\x80\\xc0\\x80"', b"\xe2\x82a": b'"\\xe2\\x82a"',
             "\u180f\u08c8".encode(): b'"\\u180f\\u08c8"'}
    for s, want in cases.items():
        assert go_quote_ref(s) == want, s


def test_quote_every_scalar_value(oracle):
    cps = scalars()
    quoters = {"oracle obo_quote": oracle.quote, "product hs_go_quote": hostsim.go_quote}
    for k in range(0, len(cps), 4096):
        s = "".join(map(chr, cps[k:k + 4096].tolist())).encode("utf-8")
        want = go_quote_ref(s)
        for who, q in quoters.items():
            got = q(s)
            if got != want:
                bad = [int(c) for c in cps[k:k + 4096] if q(chr(c).encode()) != go_quote_ref(chr(c).encode())]
                pytest.fail(f"{who} quotes {len(bad)} code points unlike Go 1.16: {cp_list(bad)}")


def test_quote_invalid_utf8(oracle):
    pieces = LONE + INVALID + [p + t for p in INVALID for t in (b"a", "\u00e9".encode(), b"\x80", b"\"")]
    pieces += [bytes([a, b]) for a in range(0x80, 0x100) for b in (0x41, 0x80, 0xBF, 0xC3)]
    for p in pieces:
        want = go_quote_ref(p)
        assert oracle.quote(p) == want, p
        assert hostsim.go_quote(p) == want, p


# ---------------------------------------------------------------------------------------------------------------------
# 4. the sweep
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def sweep():
    """(data uint8, doc_off uint64[ndocs+1], {context: slice of the documents}): every scalar value X in the five contexts,
    then every two-byte string whose first byte is >= 0x80 and every invalid pattern in `marker`, `value` and `bool`"""
    xs = [chr(c).encode("utf-8") for c in scalars().tolist()]
    extra = [bytes([a, b]) for a in range(0x80, 0x100) for b in range(256)] + INVALID
    parts, lens, spans = [], [], {}
    for name, (pre, post) in CONTEXTS.items():
        spans[name] = slice(len(lens), len(lens) + len(xs))
        parts += [pre + x + post for x in xs]
        lens += [len(pre) + len(x) + len(post) for x in xs]
    for name in ("marker", "value", "bool"):
        pre, post = CONTEXTS[name]
        spans[name + "+extra"] = slice(len(lens), len(lens) + len(extra))
        parts += [pre + x + post for x in extra]
        lens += [len(pre) + len(x) + len(post) for x in extra]
    data = np.frombuffer(b"".join(parts), dtype=np.uint8)
    off = np.zeros(len(lens) + 1, dtype=np.uint64)
    off[1:] = np.cumsum(lens)
    return data, off, spans


@functools.lru_cache(maxsize=None)
def oracle_sweep():
    import oracle
    data, off, _ = sweep()
    return oracle.lex_batch_raw(data, off)


def first_diff(a, aoff, b, boff):
    """index of the first document whose serialised stream differs (None: equal)"""
    if a == b and np.array_equal(aoff, boff):
        return None
    d = np.flatnonzero(aoff != boff)
    first = int(d[0]) - 1 if len(d) else len(aoff) - 2
    va, vb = np.frombuffer(a, np.uint8), np.frombuffer(b, np.uint8)
    n = min(len(va), len(vb))
    m = np.flatnonzero(va[:n] != vb[:n])
    if len(m):
        first = min(first, int(np.searchsorted(aoff, m[0], side="right")) - 1)
    return max(first, 0)


def assert_same_streams(got, got_off, want, want_off, what):
    d = first_diff(got, got_off, want, want_off)
    if d is not None:
        import oracle
        data, off, _ = sweep()
        doc = data[int(off[d]):int(off[d + 1])].tobytes()
        g = oracle.parse_stream(got[int(got_off[d]):int(got_off[d + 1])])
        w = oracle.parse_stream(want[int(want_off[d]):int(want_off[d + 1])])
        pytest.fail(f"{what}: document {d} {doc!r} differs from the oracle:\n got  {g}\n want {w}")


def record_flags(stream, soff):
    """per document of a serialised batch: which lexeme types it holds (bool[ndocs, 21]) and whether it holds an Error
    lexeme of the lexer's numeric check ("invalid integer literal" / "invalid float literal")"""
    s = np.frombuffer(stream, np.uint8)
    pos, end = soff[:-1].astype(np.int64), soff[1:].astype(np.int64)
    has = np.zeros((len(pos), 21), dtype=bool)
    numerr = np.zeros(len(pos), dtype=bool)
    while True:
        act = np.flatnonzero(pos < end)
        if not len(act):
            return has, numerr
        p = pos[act]
        t = s[p].astype(np.int64)
        vlen = s[p + 9].astype(np.int64) | s[p + 10].astype(np.int64) << 8 | s[p + 11].astype(np.int64) << 16 | s[p + 12].astype(np.int64) << 24
        has[act, t] = True
        e = (t == 0) & (vlen >= 9)
        if e.any():
            q = p[e] + 13
            head = np.stack([s[q + k] for k in range(9)], axis=1)
            numerr[act[e]] |= (head[:, :8] == np.frombuffer(b"invalid ", np.uint8)).all(axis=1) & np.isin(head[:, 8], [ord("i"), ord("f")])
        pos[act] = p + 13 + vlen


def assert_class_consequences(stream, soff):
    """what the lexer must do with each scalar X, from the fixture alone"""
    _data, _off, spans = sweep()
    cps = scalars()
    has, numerr = record_flags(stream, soff)
    rules = [("marker", "a MarkerStart after '+'", has[:, 2], member("letter")[cps]),
             ("value", "a number (Int / Float lexeme or a numeric literal error)", has[:, 9] | has[:, 10] | numerr,
              member("number")[cps] | np.isin(cps, [ord("."), ord("-")])),
             ("bool", "a BoolLiteral after X", has[:, 12], member("space")[cps])]
    errors = []
    for ctx, what, got, want in rules:
        bad = cps[got[spans[ctx]] != want]
        if len(bad):
            pre, post = CONTEXTS[ctx]
            errors.append(f"{pre.decode()}X{post.decode()}: {what} for {len(bad)} X against Unicode 13.0: {cp_list(bad)}")
    assert not errors, "\n".join(errors)


def test_sweep_host_core_equals_oracle(oracle):
    data, off, _ = sweep()
    want, want_off, want_n = oracle_sweep()
    got, got_off, got_n = hostsim.lex_decode_batch(data, off)
    assert_same_streams(got, got_off, want, want_off, "host core + decoder")
    assert np.array_equal(got_n, want_n)


def test_sweep_class_consequences(oracle):
    want, want_off, _ = oracle_sweep()
    assert_class_consequences(want, want_off)


# ---------------------------------------------------------------------------------------------------------------------
# 5. parser messages
# ---------------------------------------------------------------------------------------------------------------------
F = b"+operator-builder:field"


def typed_doc(x: bytes) -> bytes:
    return b"# +operator-builder:field:name=x,type=a" + x + b"\n"


def test_parser_messages_quote_like_go(oracle):
    from oracle import parser_oracle as po
    from tests import typed_parser_oracle as tpo
    rng = random.Random(13)
    cps = scalars()
    sample = sorted(set(rng.sample(cps.tolist(), 3000)) | set(range(0x80)))
    spaces = np.flatnonzero(member("space")).tolist()
    names = hostsim.Registry({b"+a": [b"b"]})
    for c in spaces + sample:
        for lit in (b"true", b"false"):
            doc = b"+a:b=" + chr(c).encode() + lit
            want = po.serialize(po.parse(oracle.lex(doc), {b"+a": {b"b"}}))
            got = hostsim.parse_doc(names, doc)
            if member("space")[c]:  # ParseBool of the whole bool literal, quoted as Go quotes it
                assert b"strconv.ParseBool: parsing " + go_quote_ref(chr(c).encode() + lit) + b": invalid syntax" in got, (f"U+{c:04X}", got)
            assert got == want, (f"U+{c:04X}", doc, want)
    typed = hostsim.Registry(define=[0])  # OBM_FIELD_MARKER
    spec = {F: tpo.OPERATOR_BUILDER_TYPED[F]}
    bmp = cps[cps < 0x10000]
    for c in bmp[~member("print")[bmp]].tolist() + sample:
        doc = typed_doc(chr(c).encode())
        want = tpo.serialize(tpo.parse(oracle.lex(doc), spec))
        got = hostsim.parse_doc(typed, doc)
        if c != 0x0A and not member("print")[c]:  # no delimiter but '\n' is unprintable: the value is "a" + X
            assert b"unable to unmarshal arg value " + go_quote_ref(b"a" + chr(c).encode()) + b", unable to parse field" in got, (f"U+{c:04X}", got)
        assert got == want, (f"U+{c:04X}", doc, want)


# ---------------------------------------------------------------------------------------------------------------------
# 6-8. GPU: the sweep through every scan mode, the device entry point, the device hash; obm_parse_batch
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scanner():
    import operator_builder_b200 as ob
    sc = ob.Scanner(0)
    yield sc
    sc.set_mode(0)
    sc.close()


@pytest.mark.gpu
def test_sweep_gpu_every_mode(scanner, oracle):
    import torch
    from operator_builder_b200 import _native
    data, off, _ = sweep()
    want, want_off, want_n = oracle_sweep()
    ndocs = len(off) - 1
    scanner.set_mode(0)
    ref = scanner.lex_batch(data, off)
    assert ref.stats["n_lexemes"] == int(want_n.sum())
    for mode in (1, 2, 3):
        scanner.set_mode(mode)
        res = scanner.lex_batch(data, off)
        assert res.stats["n_lexemes"] == int(want_n.sum()), mode
        assert np.array_equal(res.doc_tuple_off, ref.doc_tuple_off), mode
        if not np.array_equal(res.tuples, ref.tuples):
            d = int(np.searchsorted(ref.doc_tuple_off, np.flatnonzero(res.tuples != ref.tuples)[0], side="right")) - 1
            pytest.fail(f"mode {mode}: the tuples of document {d} {data[int(off[d]):int(off[d + 1])].tobytes()!r} differ from mode 0")
        del res
    scanner.set_mode(0)
    got, got_off = hostsim.decode_batch(data, off, ref.tuples, ref.doc_tuple_off)
    assert_same_streams(got, got_off, want, want_off, "mode 0, decoded")
    assert_class_consequences(got, got_off)

    # mode 0 once more through the device entry point, the batch at byte offset 7 of its buffer
    buf = torch.zeros(len(data) + 256, dtype=torch.uint8, device="cuda:0")
    buf[7:7 + len(data)] = torch.from_numpy(data.copy()).to("cuda:0")
    d_off = torch.from_numpy(off.view(np.int64).copy()).to("cuda:0")
    cap = len(ref.tuples) + 64
    d_out = torch.full((cap,), -1, dtype=torch.int64, device="cuda:0")
    d_toff = torch.zeros(ndocs + 1, dtype=torch.int64, device="cuda:0")
    d_status = torch.zeros(4, dtype=torch.int32, device="cuda:0")
    stream = torch.cuda.current_stream().cuda_stream
    scanner.lex_batch_device(buf.data_ptr() + 7, d_off.data_ptr(), ndocs, len(data), d_out.data_ptr(), cap, d_toff.data_ptr(),
                             d_status.data_ptr(), None, stream)
    torch.cuda.synchronize()
    status = d_status.cpu().tolist()
    assert status[0] == 0 and status[3] == 0, status
    assert np.array_equal(d_toff.cpu().numpy().view(np.uint64), ref.doc_tuple_off)
    assert np.array_equal(d_out.cpu().numpy().view(np.uint64)[:len(ref.tuples)], ref.tuples)

    # obm_hash_batch_device over the same stream: every nonzero hash is the oracle's, the zeros are what it leaves the host
    d_bytes = torch.zeros(len(data) + 64, dtype=torch.uint8, device="cuda:0")
    d_bytes[:len(data)] = buf[7:7 + len(data)]
    d_tup = torch.from_numpy(ref.tuples.view(np.int64).copy()).to("cuda:0")
    d_hash = torch.full((ndocs + 8,), 0x1234, dtype=torch.int64, device="cuda:0")
    d_nh = torch.full((1,), 77, dtype=torch.int32, device="cuda:0")
    rc = _native.lib().obm_hash_batch_device(scanner.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, d_tup.data_ptr(),
                                             d_toff.data_ptr(), d_hash.data_ptr(), d_nh.data_ptr(), stream)
    assert rc == 0
    torch.cuda.synchronize()
    h = d_hash.cpu().numpy().view(np.uint64)
    assert (h[ndocs:] == 0x1234).all()
    h = h[:ndocs]
    _nl, _nm, _h, want_h = oracle.scan_batch(data, off, 8, want_doc_hash=True)
    nz = h != 0
    bad = np.flatnonzero(nz & (h != want_h))
    assert not len(bad), f"{len(bad)} device hashes differ, first document {int(bad[0])} {data[int(off[bad[0]]):int(off[bad[0] + 1])].tobytes()!r}"
    assert int(d_nh.item()) == int((~nz).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["names", "typed"])
def test_parse_batch_gpu_messages(scanner, oracle, kind):
    """obm_parse_batch over +a:b=Xtrue (names-only registry {+a: [b]}) and over type=aX (the typed field marker), every
    scalar X: each document formatted == the parser oracle"""
    import operator_builder_b200 as ob
    from oracle import parser_oracle as po
    from tests import typed_parser_oracle as tpo
    if kind == "names":
        reg, oracle_parse, spec = ob.Registry({b"+a": [b"b"]}), po, {b"+a": {b"b"}}
        docs = [b"+a:b=" + chr(c).encode() + b"true" for c in scalars().tolist()]
    else:
        reg, oracle_parse, spec = ob.Registry.define(ob.FIELD_MARKER), tpo, {F: tpo.OPERATOR_BUILDER_TYPED[F]}
        docs = [typed_doc(chr(c).encode()) for c in scalars().tolist()]
    data = np.frombuffer(b"".join(docs), dtype=np.uint8)
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    scanner.set_mode(0)
    res = scanner.parse_batch(reg, data, off)
    for i, doc in enumerate(docs):
        want = oracle_parse.serialize(oracle_parse.parse(oracle.lex(doc), spec))
        got = res.format_doc(i, doc)
        assert got == want, (f"U+{int(scalars()[i]):04X}", doc, got, want)
