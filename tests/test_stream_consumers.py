"""The device consumers of the tuple stream, each against a reference of its own.

- Value typing (ParseFloat(., 32) range, ParseBool) in obm_parse.cpp, obm_parse_dev.h (k_parse_docs) and
  oracle/parser_oracle.py, and the lexer's ParseFloat(., 64) check, against go_parse_float_range below: Go's readFloat
  restated over exact decimals.
- obm_hash_batch_device (k_hash_docs) on real tuple streams, against FNV-1a over the decoded stream and the oracle's
  per-document hash; both of its paths (a group's tuples staged in shared memory or read from global memory).
- obm_marker_index_flat_device (k_marker_index_flat) at its tile edges, against the per-document index and the parser
  oracle's loaded definitions.
- obm_lex_batch_device with a batch that does not start on a 16-byte boundary.
"""
import random
import re
from decimal import Decimal

import numpy as np
import pytest

from tests import corpus_util as cu
from tests import hostsim
from tests import test_parser_row as tpr

# ---------------------------------------------------------------------------------------------------------------------
# 1. Go's numeric checks
# ---------------------------------------------------------------------------------------------------------------------
# the smallest magnitudes that round (half to even) to +Inf: the largest finite value plus half an ULP
F32_LIMIT = Decimal(2 ** 128 - 2 ** 103)
F64_LIMIT = Decimal(2 ** 1024 - 2 ** 970)
_DECIMAL = re.compile(rb"[+-]?([0-9]*)(?:\.([0-9]*))?(?:[eE]([+-]?)([0-9]+))?")


def go_parse_float_range(s: bytes, bits: int) -> int:
    """Error class of strconv.ParseFloat(s, bits) for decimal input: 0 ok, 1 invalid syntax, 2 value out of range.
    Go's readFloat stops accumulating exponent digits once the exponent reaches 10000 (it is then only a bound on how
    far the point moves), so the literal means digits * 10**(saturated exponent - fraction digits); that Decimal is
    exact for any number of digits, and so is its comparison with the limit."""
    m = _DECIMAL.fullmatch(s)
    if m is None or not (m.group(1) or m.group(2)):
        return 1
    whole, frac, esign, edigits = m.group(1), m.group(2) or b"", m.group(3), m.group(4) or b""
    e = 0
    for ch in edigits:
        if e < 10000:
            e = e * 10 + ch - 0x30
    if esign == b"-":
        e = -e
    mant = (whole + frac).lstrip(b"0")
    if not mant:
        return 0
    value = Decimal(f"{mant.decode()}E{e - len(frac)}")
    return 2 if value >= (F32_LIMIT if bits == 32 else F64_LIMIT) else 0


GO_PARSE_BOOL = {b"1", b"t", b"T", b"TRUE", b"true", b"True", b"0", b"f", b"F", b"FALSE", b"false", b"False"}  # strconv/atob.go


def _sci(digits: str, extra: str = "", exp_fmt="e{}", lead="") -> bytes:
    """digits (the integer value) + extra fraction digits, written as d.ddd...e<len-1>"""
    return f"{lead}{digits[0]}.{digits[1:]}{extra}{exp_fmt.format(len(digits) - 1)}".encode()


def numeric_cases():
    t32, t64 = str(2 ** 128 - 2 ** 103), str(2 ** 1024 - 2 ** 970)
    out = [b"3.4028235e38", b"3.4028236e38", b"3.40282356779733661637539395458142568447e38", b"1e39", b"1e38",
           b"1.7976931348623157e308", b"1.7976931348623159e308", b"1e308", b"1e309"]
    for t in (t32, t64):
        below = str(int(t) - 1)
        for d in (t, below):
            out += [d.encode() + b".", d.encode() + b".0", _sci(d), _sci(d, lead="-"), b"." + d.encode() + b"e%d" % len(d),
                    b"0.000" + d.encode() + b"e%d" % (len(d) + 3), b"000" + d.encode() + b".000", _sci(d, exp_fmt="e+{:04d}"),
                    _sci(d, exp_fmt="E{:05d}"), b"-0.0" + d.encode() + b"e%d" % (len(d) + 1)]
        for k in range(1, 61):  # the threshold, then k more digits: zeros and a final 1; below it, nines
            out += [_sci(t, "0" * (k - 1) + "1"), _sci(t, "0" * k), _sci(below, "9" * k),
                    b"0." + t.encode() + b"0" * (k - 1) + b"1e%d" % len(t)]
        # one unit below / above in the last digit, with the point elsewhere
        out += [(below[:10] + "." + below[10:]).encode() + b"e%d" % (len(t) - 10), (t[:10] + "." + t[10:]).encode() + b"e%d" % (len(t) - 10)]
    # exponents of 4 to 7 digits on both sides of the saturation at 10000: 0.(k zeros)1eE = 10**(sat(E) - k - 1)
    for edig, sat in ((b"9999", 9999), (b"10000", 10000), (b"10001", 10000), (b"99999", 10000), (b"100000", 10000),
                      (b"1000000", 10000), (b"0010000", 10000), (b"00009999", 9999), (b"9999999", 99999)):
        for lim in (39, 309):
            for k in (sat - lim - 1, sat - lim):
                out += [b"0." + b"0" * k + b"1e" + edig, b"-0." + b"0" * k + b"1e" + edig]
        out += [b"1e" + edig, b"1e-" + edig, b"1." + b"e" + edig]
    # long mantissas (4,300 digits is Python's int-string limit); the point stays within the first 800 digits, where
    # Go's decimal fallback reads the same value (DESIGN.md, "Parity unpinned")
    for n in (4299, 4301, 20000, 100000):
        out += [t32.encode() + b"." + b"0" * (n - 39), str(int(t32) - 1).encode() + b"." + b"9" * (n - 39),
                t64.encode() + b"." + b"0" * (n - 309), str(int(t64) - 1).encode() + b"." + b"9" * (n - 309),
                b"1" * n + b"e-%d" % (n - 37), b"0." + b"0" * n + b"1e%d" % min(n, 9999), b"9" * n + b"." + b"5"]
    out.append(b"0." + b"0" * 20000 + b"1e100000")  # reads as 1e-10001: in range, though the exact value is 1e79999
    out += [b"1e-400", b"1e-46", b"-1e-400", b"0.0000000000000000000000000000000000000000000001", b"1e-99999", b"0e99999", b"-0.0e400"]
    return out


def bool_cases():
    return sorted(GO_PARSE_BOOL) + [b"tRUE", b"TRUe", b"True ", b" true", b"2", b"", b"yes", b"t ", b"FaLsE", b"fALSE", b"truE",
                                    b"00", b"10", b"tr", b"TR", b"Fals", b"falsee", b"\ttrue"]


def test_reference_itself():
    """known values of Go's strconv, and the readFloat saturation"""
    r = go_parse_float_range
    assert r(b"3.4028235e38", 32) == 0 and r(b"3.4028236e38", 32) == 2 and r(b"340282356779733661637539395458142568448.", 32) == 2
    assert r(b"340282356779733661637539395458142568447.9", 32) == 0
    assert r(b"1.7976931348623157e308", 64) == 0 and r(b"1.7976931348623159e308", 64) == 2
    assert r(b"1e-400", 64) == 0 and r(b".", 64) == 1 and r(b"1e", 64) == 1 and r(b"1.", 64) == 0 and r(b".5", 64) == 0
    assert r(b"0." + b"0" * 20000 + b"1e100000", 32) == 0 and r(b"0." + b"0" * 9960 + b"1e100000", 32) == 2
    assert r(b"0." + b"0" * 9961 + b"1e100000", 32) == 0


def test_parser_oracle_reads_every_literal():
    """parser_oracle's ParseFloat(., 32) range is readFloat's: exact, saturated, for any number of digits"""
    from oracle import parser_oracle as po
    for s in numeric_cases():
        if go_parse_float_range(s, 64) == 1:
            continue
        assert (po.read_float_magnitude(s) >= po.F32_OVERFLOW_DEC) == (go_parse_float_range(s, 32) == 2), s[:80]


def test_float64_range_matches_reference(oracle):
    """the lexer's ParseFloat(., 64): the oracle's C restatement and the product's (obm_core.h parse_float_err)"""
    L, H = oracle.lib(), hostsim.lib()
    for s in numeric_cases():
        want = go_parse_float_range(s, 64)
        assert L.obo_parse_float_err(s, len(s)) == want, s[:80]
        assert H.hs_parse_float_err(s, len(s)) == want, s[:80]


def _in_lexer_alphabet(s):
    """literals the lexer reads whole as one FloatLiteral (lexNumericLiteral: '.', '-' or a digit first, then digits,
    '.', 'e', 'E', '-'; a '.', 'e' or '-' after the first byte makes it a float)"""
    return bool(s) and s[:1] in b".-0123456789" and all(c in b"0123456789.eE-" for c in s) and (s[:1] == b"." or any(c in b".eE-" for c in s[1:]))


def marker_doc(lit: bytes) -> bytes:
    return b"# +operator-builder:field:name=x,default=" + lit + b"\n"


def expect_marker(lit: bytes):
    """what parser.Parse must return for marker_doc(lit): ('lexer', ...) when the lexer rejects the literal
    (ParseFloat(., 64), state.go:258), ('range', ...) for ParseFloat(., 32) out of range, else ('ok', ...)"""
    if go_parse_float_range(lit, 64):
        return "lexer"
    return "range" if go_parse_float_range(lit, 32) else "ok"


def outcome(results, value: bytes):
    """category of a parser_oracle result list for one marker whose `default` carries `value`"""
    assert len(results) == 1, results
    r = results[0]
    if r[0] == "ok":
        assert (b"default", "float", value) in r[3] or (b"default", "bool", value) in r[3], r
        return "ok"
    if r[1].startswith("invalid float literal"):
        return "lexer"
    if "value out of range" in r[1]:
        return "range"
    if "invalid syntax" in r[1] and r[1].startswith("strconv.ParseBool"):
        return "bool"
    raise AssertionError(r)


def test_float32_range_through_markers(oracle):
    """every literal the lexer reads whole, as the `default` of a field marker: obm_parse_doc, the device walk on the
    host and parser_oracle agree byte for byte, and on the outcome the reference gives"""
    from oracle import parser_oracle as po
    n = 0
    for lit in numeric_cases():
        if not _in_lexer_alphabet(lit):
            continue
        doc = marker_doc(lit)
        tpr.check(oracle, doc)
        got = outcome(po.parse(oracle.lex(doc), po.OPERATOR_BUILDER_REGISTRY), lit)
        assert got == expect_marker(lit), lit[:80]
        n += 1
    assert n > 300


def synthetic(value: bytes, kind: int, oracle):
    """a field marker whose `default` value lexeme is `value` with the given kind, whatever the lexer would make of
    those bytes: the document is lexed with a placeholder naked string of the same length, whose tuple (and oracle
    lexeme) then take the kind, and whose bytes are replaced.  -> (doc, tuples, oracle lexemes)"""
    ph = b"a" * max(1, len(value))
    doc0 = b"+operator-builder:field:default=" + ph + b"\n"
    tup = hostsim.lex_doc(doc0).copy()
    kinds = tup >> np.uint64(59)
    (k,) = np.nonzero(kinds == 8)[0]
    off = int(tup[k] & np.uint64(0xFFFFFFFF))
    tup[k] = np.uint64((kind << 59) | (len(value) << 32) | off)
    doc = doc0[:off] + value + b"\x00" * (len(ph) - len(value)) + doc0[off + len(ph):]
    lx = oracle.lex(doc0)
    (j,) = [i for i, x in enumerate(lx) if x[0] == 8]
    lx[j] = (kind, value, lx[j][2], lx[j][3])
    return doc, tup, lx


def test_value_typing_on_synthetic_lexemes(oracle):
    """ParseFloat(., 32) and ParseBool on any value the parser can be handed, including spellings the lexer never
    produces (exponent '+', '+' sign, ParseBool near misses): three restatements, one reference"""
    from oracle import parser_oracle as po
    cases = [(v, 9) for v in numeric_cases() if go_parse_float_range(v, 64) == 0] + [(v, 12) for v in bool_cases()]
    for value, kind in cases:
        doc, tup, lx = synthetic(value, kind, oracle)
        want_bytes = po.serialize(po.parse(lx, po.OPERATOR_BUILDER_REGISTRY))
        assert tpr.results_via_tuples(doc, tup) == want_bytes, value[:80]
        assert tpr.results_via_device_walk(doc, tup) == want_bytes, value[:80]
        got = outcome(po.parse(lx, po.OPERATOR_BUILDER_REGISTRY), value)
        if kind == 9:
            assert got == ("range" if go_parse_float_range(value, 32) else "ok"), value[:80]
        else:
            assert got == ("ok" if value in GO_PARSE_BOOL else "bool"), value


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def pack(docs):
    data = np.frombuffer(b"".join(docs) + b"\0", dtype=np.uint8)[:-1] if docs else np.zeros(0, np.uint8)
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    if docs:
        off[1:] = np.cumsum([len(d) for d in docs])
    return data, off


def to_dev(a, pad=64):
    import torch
    a = np.ascontiguousarray(a)
    if a.dtype == np.uint8:
        a = np.concatenate([a, np.zeros(pad, np.uint8)])
    elif a.dtype == np.uint64:
        a = a.view(np.int64)
    return torch.from_numpy(a.copy()).to("cuda:0")


@pytest.fixture(scope="module")
def scanner():
    import operator_builder_b200 as ob
    sc = ob.Scanner(0)
    yield sc
    sc.set_mode(0)
    sc.close()


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


# ---------------------------------------------------------------------------------------------------------------------
# 1 (GPU). the lexer's float check in every mode, and k_parse_docs' value typing
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_numeric_typing_on_gpu(scanner, oracle):
    import torch
    import operator_builder_b200 as ob
    from operator_builder_b200 import _native
    from oracle import parser_oracle as po
    lits = [s for s in numeric_cases() if _in_lexer_alphabet(s)]
    docs = [marker_doc(s) for s in lits]
    data, off = pack(docs)
    streams = []
    for mode in (0, 1, 2, 3):
        scanner.set_mode(mode)
        res = scanner.lex_batch(data, off)
        streams.append(res)
        for i, lit in enumerate(lits):
            kinds = res.tuples[int(res.doc_tuple_off[i]):int(res.doc_tuple_off[i + 1])] >> np.uint64(59)
            lexed = "err" if (kinds == 30).any() else "float" if (kinds == 9).any() else "other"
            assert lexed == ("err" if go_parse_float_range(lit, 64) else "float"), (mode, lit[:80])
    scanner.set_mode(0)
    for r in streams[1:]:
        assert np.array_equal(r.tuples, streams[0].tuples) and np.array_equal(r.doc_tuple_off, streams[0].doc_tuple_off)
    # the real documents' tuples, then the synthetic lexemes (spellings the lexer never produces), as one batch
    all_docs, all_tup, lexemes = list(docs), [streams[0].tuples[int(streams[0].doc_tuple_off[i]):int(streams[0].doc_tuple_off[i + 1])]
                                              for i in range(len(docs))], [oracle.lex(d) for d in docs]
    for value, kind in [(v, 9) for v in numeric_cases() if go_parse_float_range(v, 64) == 0] + [(v, 12) for v in bool_cases()]:
        d, t, lx = synthetic(value, kind, oracle)
        all_docs.append(d); all_tup.append(t); lexemes.append(lx)
    data, off = pack(all_docs)
    toff = np.zeros(len(all_docs) + 1, np.uint64)
    toff[1:] = np.cumsum([len(t) for t in all_tup])
    tuples = np.concatenate(all_tup)
    d_bytes, d_off, d_tup, d_toff = to_dev(data), to_dev(off), to_dev(tuples), to_dev(toff)
    L = _native.lib()
    reg = tpr.REG()
    n = len(all_docs)

    def run(res_cap, arg_cap, doc_base, slack=64):
        d_res = torch.full(((res_cap + slack) * 32,), 0xA5, dtype=torch.uint8, device="cuda:0")
        d_args = torch.full(((arg_cap + slack) * 16,), 0x5A, dtype=torch.uint8, device="cuda:0")
        d_roff = torch.zeros(n + 1, dtype=torch.int64, device="cuda:0")
        d_tot = torch.full((2,), -1, dtype=torch.int64, device="cuda:0")
        rc = L.obm_parse_batch_device(scanner.handle, reg.handle, d_bytes.data_ptr(), d_off.data_ptr(), n, doc_base, d_tup.data_ptr(),
                                      d_toff.data_ptr(), d_res.data_ptr(), res_cap, d_args.data_ptr(), arg_cap, d_roff.data_ptr(),
                                      d_tot.data_ptr(), _stream())
        assert rc == 0
        torch.cuda.synchronize()
        return d_res.cpu().numpy(), d_args.cpu().numpy(), d_roff.cpu().numpy(), [int(x) for x in d_tot.cpu().tolist()]

    big = len(tuples) + 8
    R8, A8, roff, (nres, nargs) = run(big, big, 7000)
    assert nres == int(roff[-1])
    R, A = R8[:nres * 32].view(tpr.RES_DT), A8[:nargs * 16].view(tpr.ARG_DT)
    host = 0
    for i, doc in enumerate(all_docs):
        r = R[int(roff[i]):int(roff[i + 1])]
        assert all(int(x) == i + 7000 for x in r["doc"])
        host += int(len(r) == 1 and int(r[0]["flags"]) & tpr.R_HOST != 0)
        got = tpr.format_records(doc, all_tup[i], r, A)
        want = po.serialize(po.parse(lexemes[i], po.OPERATOR_BUILDER_REGISTRY))
        assert got == want, (i, doc[:120])
        if i < len(lits):
            assert outcome(po.parse(lexemes[i], po.OPERATOR_BUILDER_REGISTRY), lits[i]) == expect_marker(lits[i])
    assert host <= len(lits) // 2  # the lexer-error documents go back to the host; the typed values are the device's
    # capacities below the totals: the totals stay whole and nothing lands past either capacity
    rc_, ac_ = nres - 5, nargs - 3
    R8c, A8c, roffc, tot = run(rc_, ac_, 123456)
    assert tot == [nres, nargs] and np.array_equal(roffc, roff)
    assert (R8c[rc_ * 32:] == 0xA5).all() and (A8c[ac_ * 16:] == 0x5A).all()
    Rc = R8c[:rc_ * 32].view(tpr.RES_DT).copy()
    Rc["doc"] -= 123456 - 7000
    assert np.array_equal(Rc, R[:rc_]) and np.array_equal(A8c[:ac_ * 16], A8[:ac_ * 16])


# ---------------------------------------------------------------------------------------------------------------------
# 2. obm_hash_batch_device on real streams
# ---------------------------------------------------------------------------------------------------------------------
_FNV_PRIME, _MASK = 0x100000001B3, (1 << 64) - 1


def fnv1a(b: bytes) -> int:
    h = 0xCBF29CE484222325
    for c in b:
        h = ((h ^ c) * _FNV_PRIME) & _MASK
    return h


def host_flag(doc: bytes, t: np.ndarray) -> bool:
    """the documents the device hash leaves to the host: a pseudo-tuple other than LINE, or a byte >= 0x80 inside the
    value of a lexeme that takes its value from the document (not SyntheticBool / MarkerEnd / EOF)"""
    k = (t >> np.uint64(59)).astype(np.int64)
    if ((k > 20) & (k != 24)).any():
        return True
    sliced = (k >= 1) & (k <= 13) & (k != 11)
    off = (t & np.uint64(0xFFFFFFFF)).astype(np.int64)[sliced]
    ln = ((t >> np.uint64(32)) & np.uint64((1 << 27) - 1)).astype(np.int64)[sliced]
    hi = np.concatenate([[0], np.cumsum(np.frombuffer(doc, np.uint8) >= 0x80)])
    return bool((hi[off + ln] - hi[off] > 0).any())


def hash_and_check(scanner, oracle, docs, min_device_share=None):
    """scan (mode 0), hash on the device, and check every document -> (tuples per document, flagged count)"""
    import torch
    import operator_builder_b200 as ob
    from operator_builder_b200 import _native
    scanner.set_mode(0)
    data, off = pack(docs)
    res = scanner.lex_batch(data, off)
    n = len(docs)
    d_bytes, d_off, d_tup, d_toff = to_dev(data), to_dev(off), to_dev(res.tuples), to_dev(res.doc_tuple_off)
    d_hash = torch.full((n + 8,), 0x1234, dtype=torch.int64, device="cuda:0")
    d_nh = torch.full((1,), 77, dtype=torch.int32, device="cuda:0")
    rc = _native.lib().obm_hash_batch_device(scanner.handle, d_bytes.data_ptr(), d_off.data_ptr(), n, d_tup.data_ptr(), d_toff.data_ptr(),
                                             d_hash.data_ptr(), d_nh.data_ptr(), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    got = d_hash.cpu().numpy().view(np.uint64)
    assert (got[n:] == 0x1234).all()
    _nl, _nm, _h, want = oracle.scan_batch(data if len(data) else np.zeros(1, np.uint8), off, 4, want_doc_hash=True)
    flagged = 0
    for i, doc in enumerate(docs):
        t = res.tuples[int(res.doc_tuple_off[i]):int(res.doc_tuple_off[i + 1])]
        if host_flag(doc, t):
            flagged += 1
            assert int(got[i]) == 0, (i, doc[:100])
        else:
            h = fnv1a(ob.decode_doc_raw(doc, t))
            assert int(got[i]) == h == int(want[i]), (i, doc[:100], int(got[i]), h, int(want[i]))
    assert int(d_nh.item()) == flagged
    if min_device_share is not None:
        assert n - flagged >= min_device_share * n, (flagged, n)
    return np.diff(res.doc_tuple_off.astype(np.int64)), flagged


@pytest.mark.gpu
def test_hash_on_real_corpora(scanner, oracle):
    import json
    import os
    golden = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "lexer_golden.json")))
    rng = random.Random(2024)
    hash_and_check(scanner, oracle, [c["input"].encode() for c in golden["cases"]])
    hash_and_check(scanner, oracle, list(cu.TARGETED))
    _, fl = hash_and_check(scanner, oracle, list(cu.NON_ASCII))
    assert fl > 0
    hash_and_check(scanner, oracle, [d for _p, d in cu.fixtures()], min_device_share=0.6)
    hash_and_check(scanner, oracle, [cu.fuzz_doc(rng, max_len=400, non_ascii=k % 2 == 1) for k in range(3000)])
    hash_and_check(scanner, oracle, [cu.fuzz_doc_valid(rng) for _ in range(1000)])  # most of these hold a PART or a warning
    hash_and_check(scanner, oracle, [cu.fuzz_doc_valid(rng, max_lines=2) for _ in range(2000)], min_device_share=0.6)
    import operator_builder_b200 as ob
    for flavour in (0, 1):
        data0, _ = ob.generate_corpus_host(200, 4096, flavour=flavour)
        hash_and_check(scanner, oracle, [data0.tobytes()[i * 4096:(i + 1) * 4096] for i in range(200)], min_device_share=1.0)


@pytest.mark.gpu
def test_hash_on_large_documents_and_sweep(scanner, oracle):
    """the large-document corpus and the adversarial sweep cells of test_gpu_parity.py"""
    rng = random.Random(11)
    big = []
    for target in (1 << 20, 3 << 20):
        parts, n = [], 0
        while n < target:
            ln = rng.choice([b"key: value\n", b"  - item  # +operator-builder:field:name=a.b,type=int,default=3\n", b"\n",
                             b"# +x:y=`multi\n  # line`\n", b"path: /a/b+c\n", b"x" * 300 + b"\n"])
            parts.append(ln)
            n += len(ln)
        big.append(b"".join(parts))
    counts, _ = hash_and_check(scanner, oracle, big + [b"+a:b"] + big[:1] + ["# é +a:b=ü\n".encode() * 2500])
    assert counts[0] > 6144  # a group read from global memory
    docs = []
    for m in (0, 1, 2, 4, 8, 16, 32, 64):
        for L in (16, 64, 256, 1024, 4096, 16384, 65536):
            line = b"# " + b" ".join(b"+s:a%d=%d" % (k, k) for k in range(m))
            if len(line) + 1 > L:
                line = line[:L - 1]
            pad = L - 1 - len(line)
            variants = [line + b" " + b"x" * (pad - 1) if pad > 0 else line,
                        line + (b" +q:v=\"" + b"y" * (pad - 9) + b"\"" if pad > 9 else b" " * pad),
                        line + (b" +q:v=" + b"z" * (pad - 6) if pad > 6 else b" " * pad)]
            for v in variants:
                docs.append((v + b"\n") * max(1, min(8, 131072 // L)))
    hash_and_check(scanner, oracle, docs)


@pytest.mark.gpu
def test_hash_staging_boundary_and_ragged_batches(scanner, oracle):
    """k_hash_docs stages a group of 32 documents in shared memory when its tuples fit in PD_CAP = 6,144 and reads
    global memory otherwise: groups of exactly 6,144 and 6,145 tuples, and batches of 1, 31, 33 and 77 documents"""
    rng = random.Random(9)
    pool = [cu.fuzz_doc_valid(rng, max_lines=300) for _ in range(300)] + [d for _p, d in cu.fixtures()]
    fillers = [b"# c\n" * k for k in range(1, 2000)] + [b"k: v\n" + b"# c\n" * k for k in range(0, 2000)]
    data, off = pack([b""] + pool + fillers)
    counts = np.diff(scanner.lex_batch(data, off).doc_tuple_off.astype(np.int64))
    assert counts[0] == 1  # an empty document is one EOF
    pc, fc = counts[1:1 + len(pool)], counts[1 + len(pool):]
    by_count = {}
    for f, c in zip(fillers, fc):
        by_count.setdefault(int(c), f)
    assert all(c in by_count for c in range(1, 3999))
    batch, targets = [], [6144, 6145, 6144, 6145, 6143, 6144]
    for target in targets:  # pool documents while the rest exceeds what one filler holds, empty documents, one filler
        idx, s = [], 0
        for i in rng.sample(range(len(pool)), len(pool)):
            if len(idx) == 31 or target - s - (31 - len(idx)) < 3999:
                break
            if s + int(pc[i]) + (31 - len(idx) - 1) < target:
                idx.append(i)
                s += int(pc[i])
        rest = target - s - (31 - len(idx))
        assert rest in by_count, (target, s, len(idx))
        group = [pool[i] for i in idx] + [b""] * (31 - len(idx)) + [by_count[rest]]
        rng.shuffle(group)
        batch += group
    counts, _ = hash_and_check(scanner, oracle, batch)
    assert list(counts.reshape(-1, 32).sum(axis=1)) == targets
    for n in (1, 31, 33, 77):
        hash_and_check(scanner, oracle, batch[:n])
        hash_and_check(scanner, oracle, rng.sample(pool, n))


# ---------------------------------------------------------------------------------------------------------------------
# 3. obm_marker_index_flat_device at its tile edges
# ---------------------------------------------------------------------------------------------------------------------
FI_TILE = 2048
REC_DT = np.dtype([("doc", "<u4"), ("tuple", "<u4"), ("off", "<u4"), ("reg_scopes", "<u4")])


def flat_index(scanner, registry, docs, doc_base=0, bound_extra=0, cap=None, records=True, res=None):
    """-> (records, total, rc) of obm_marker_index_flat_device; records beyond cap must stay untouched"""
    import torch
    from operator_builder_b200 import _native
    data, off = pack(docs)
    if res is None:
        res = scanner.lex_batch(data, off)
    ntup = len(res.tuples)
    d_bytes, d_off = to_dev(data), to_dev(off)
    d_tup, d_toff = to_dev(res.tuples if ntup else np.zeros(1, np.uint64)), to_dev(res.doc_tuple_off)
    cap = ntup if cap is None else cap
    d_rec = torch.full(((cap + 64) * 4,), -7, dtype=torch.int32, device="cuda:0")
    d_tot = torch.full((1,), -1, dtype=torch.int64, device="cuda:0")
    rc = _native.lib().obm_marker_index_flat_device(scanner.handle, registry.handle, d_bytes.data_ptr(), d_off.data_ptr(), len(docs), doc_base,
                                                    d_tup.data_ptr(), d_toff.data_ptr(), ntup + bound_extra,
                                                    d_rec.data_ptr() if records else None, cap, d_tot.data_ptr(), _stream())
    if rc != 0:
        return None, None, rc
    torch.cuda.synchronize()
    rec = d_rec.cpu().numpy()
    total = int(d_tot.item())
    n = min(total, cap) if records else 0
    assert (rec[n * 4:] == -7).all(), "a record past the capacity (or past the count) was written"
    return rec[:n * 4].view(np.uint32).view(REC_DT).copy(), total, 0


def per_doc_index(scanner, registry, docs, res):
    import torch
    from operator_builder_b200 import _native
    data, off = pack(docs)
    cap = max(1, len(res.tuples))
    d_bytes, d_off, d_tup, d_toff = to_dev(data), to_dev(off), to_dev(res.tuples), to_dev(res.doc_tuple_off)  # alive until synchronised
    d_rec = torch.zeros(cap * 4, dtype=torch.int32, device="cuda:0")
    d_roff = torch.zeros(len(docs) + 1, dtype=torch.int64, device="cuda:0")
    rc = _native.lib().obm_marker_index_device(scanner.handle, registry.handle, d_bytes.data_ptr(), d_off.data_ptr(), len(docs),
                                               d_tup.data_ptr(), d_toff.data_ptr(), d_rec.data_ptr(), cap, d_roff.data_ptr(), _stream())
    assert rc == 0
    torch.cuda.synchronize()
    roff = d_roff.cpu().numpy()
    return d_rec.cpu().numpy()[:int(roff[-1]) * 4].view(np.uint32).view(REC_DT).copy(), roff


def check_flat(scanner, oracle, reg_dict, docs, doc_base=0, bound_extra=0, min_records=1):
    """flat index == per-document index (+ doc_base) == the parser oracle's loaded definitions; total == count"""
    import operator_builder_b200 as ob
    from oracle import parser_oracle as po
    reg = ob.Registry(reg_dict)
    names = list(reg_dict)
    data, off = pack(docs)
    scanner.set_mode(0)
    res = scanner.lex_batch(data, off)
    flat, total, rc = flat_index(scanner, reg, docs, doc_base, bound_extra, res=res)
    assert rc == 0 and total == len(flat)
    per, roff = per_doc_index(scanner, reg, docs, res)
    want = per.copy()
    want["doc"] += doc_base
    assert np.array_equal(flat, want), (flat[:8], want[:8])
    for i, doc in enumerate(docs):
        got = per[int(roff[i]):int(roff[i + 1])]
        if not len(got) and b"+" not in doc:
            continue
        prs = po.Parser(oracle.lex(doc), reg_dict)
        prs.run()
        assert [names[int(r) & 0xFFFF] for r in got["reg_scopes"]] == prs.loaded, (i, doc[:200])
        for r in got:
            t = int(res.tuples[int(res.doc_tuple_off[i]) + int(r["tuple"])])
            assert t >> 59 == 2 and (t & 0xFFFFFFFF) == int(r["off"]) and doc[int(r["off"])] == ord("+")
    assert total >= min_records
    return res, flat


OB = {k: set(v) for k, v in {b"+operator-builder:field": [b"name", b"type", b"default"],
                             b"+operator-builder:collection:field": [b"name"], b"+operator-builder:resource": [b"field", b"include"]}.items()}
MARKER = b"# +operator-builder:field:name=x\n"


def layout(scanner, doc):
    """tuples of `doc` and the index of its first MarkerStart (measured on the device)"""
    data, off = pack([b"", doc])
    res = scanner.lex_batch(data, off)
    assert int(res.doc_tuple_off[1]) == 1, "an empty document is one EOF tuple"
    t = res.tuples[1:]
    return len(t), int(np.nonzero((t >> np.uint64(59)) == 2)[0][0])


@pytest.mark.gpu
def test_flat_index_many_documents_per_tile(scanner, oracle):
    """65, 500 and ~2,000 documents before a registered marker inside one tile: the walk past the 64 cached offsets"""
    for before in (63, 64, 65, 66, 130, 500, 1990, 2030):
        for lead in (0, 700):
            docs = [MARKER] * (lead > 0) + [b"k: v\n"] * (lead // 2) + [b""] * before + [MARKER, b"", MARKER] + [b""] * 70 + [MARKER]
            check_flat(scanner, oracle, OB, docs, doc_base=before, min_records=3)


@pytest.mark.gpu
def test_flat_index_marker_across_tiles(scanner, oracle):
    """a MarkerStart at tuple 2,044..2,047 of a tile: its Scope / Separator / Arg tuples come from the next tile"""
    n, p = layout(scanner, MARKER)
    for docs_before in ((), (MARKER,), (b"# +operator-builder:resource:field=a,include\n", b"x")):
        base = [*docs_before]
        data, off = pack(base)
        used = int(scanner.lex_batch(data, off).doc_tuple_off[-1]) if base else 0
        for target in (2044, 2045, 2046, 2047, 2048, 2 * 2048 - 1):
            pad = (target - p - used) % FI_TILE
            docs = base + [b""] * pad + [MARKER, MARKER] + [b""] * 5
            res, flat = check_flat(scanner, oracle, OB, docs, min_records=2)
            d = len(base) + pad
            assert (int(res.doc_tuple_off[d]) + p) % FI_TILE == target % FI_TILE
            assert d in set(int(x) for x in flat["doc"])
    # the last tile partly filled, and a bound several tiles above the real count
    docs = [MARKER] * 300 + [b""] * 37 + [MARKER]
    check_flat(scanner, oracle, OB, docs, bound_extra=5 * FI_TILE + 3, min_records=301)


REG8 = {b"+a:b": {b"x"}, b"+a:bb": {b"x"}, b"+a:bbb": {b"x"},                    # prefixes of each other
        b"+eq:abcd1": {b"x"}, b"+eq:abcd2": {b"x"},                              # equal length, last byte differs
        b"+long:" + b"n" * 56: {b"x"},                                           # 62 bytes: past the 48-byte vector compare
        b"+k:v:w": {b"x"}, b"+operator-builder:field": {b"name"}}


@pytest.mark.gpu
def test_flat_index_custom_registry(scanner, oracle):
    """8 names: prefixes of each other, equal lengths, one longer than 48 bytes; name starts at each offset mod 4"""
    bodies = [b"+a:b:x=1", b"+a:bb:x=1", b"+a:bbb:x", b"+a:bbbb:x=1", b"+a:bc:x=1", b"+eq:abcd1:x=1", b"+eq:abcd2:x=\"s\"", b"+eq:abcd3:x=1",
              b"+eq:abcd:x=1", b"+long:" + b"n" * 56 + b":x=1", b"+long:" + b"n" * 55 + b"m:x=1", b"+long:" + b"n" * 57 + b":x=1",
              b"+k:v:w:x=1", b"+k:v:x=1", b"+operator-builder:field:name=q", b"+operator-builder:fielD:name=q"]
    docs = []
    for pre in (b"", b"#", b"# ", b"#  "):
        for b in bodies:
            docs.append(pre + b + b"\n")
            docs.append(b"k: v\n" + pre + b + b"\n" + pre + b)
    rng = random.Random(4)
    rng.shuffle(docs)
    _res, flat = check_flat(scanner, oracle, REG8, docs, doc_base=1 << 20, min_records=96)
    assert len(set(int(x) & 0xFFFF for x in flat["reg_scopes"])) == 8
    _data, off = pack(docs)
    assert {(int(off[int(r["doc"]) - (1 << 20)]) + int(r["off"])) & 3 for r in flat} == {0, 1, 2, 3}
    # registries with more than 8 names are refused, by both indexes
    import operator_builder_b200 as ob
    reg9 = ob.Registry({**REG8, b"+z:z": {b"x"}})
    _f, _t, rc = flat_index(scanner, reg9, docs[:10])
    assert rc == -4
    data, off = pack(docs[:10])
    res = scanner.lex_batch(data, off)
    from operator_builder_b200 import _native
    import torch
    d_roff = torch.zeros(11, dtype=torch.int64, device="cuda:0")
    d_bytes, d_off, d_tup, d_toff = to_dev(data), to_dev(off), to_dev(res.tuples), to_dev(res.doc_tuple_off)
    assert _native.lib().obm_marker_index_device(scanner.handle, reg9.handle, d_bytes.data_ptr(), d_off.data_ptr(), 10, d_tup.data_ptr(),
                                                 d_toff.data_ptr(), None, 0, d_roff.data_ptr(), _stream()) == -4


@pytest.mark.gpu
def test_flat_index_stale_buffer_and_fatal_neighbours(scanner, oracle):
    """a stale '+' in the lexer's buffer (PART before the candidate) and candidates right after a document that ends in a
    fatal error, also as the first tuple of a tile"""
    stale = [b"# a+1 +operator-builder:field:name=x\n", b"++operator-builder:field:name=x", b"x+ # +operator-builder:field:name=y\n",
             b"a+b +operator-builder:field:name=z"]
    fatal = [b"# +a:b=\"unterminated\n", b"# +a:b=1e309\n", b"+a:b=99999999999999999999", b"# x+ +a:b='open", b"+a:b=,", b"a+ +c:d=\"x"]
    docs = []
    for f in fatal:
        docs += [f, b"+operator-builder:field:name=x\n", f, MARKER]
    docs += stale + [MARKER]
    check_flat(scanner, oracle, OB, docs, min_records=len(fatal) * 2)
    n, p = layout(scanner, b"+operator-builder:field:name=x\n")
    for f in fatal:  # the candidate as tuple 0 of the second tile, right after the fatal document's last tuple
        data, off = pack([f])
        nf = int(scanner.lex_batch(data, off).doc_tuple_off[-1])
        docs = [b""] * (FI_TILE - nf - p) + [f, b"+operator-builder:field:name=x\n"]
        res, flat = check_flat(scanner, oracle, OB, docs, min_records=1)
        assert int(res.doc_tuple_off[len(docs) - 1]) + p == FI_TILE


@pytest.mark.gpu
def test_flat_index_capacity_and_empty(scanner, oracle):
    import operator_builder_b200 as ob
    reg = ob.Registry(OB)
    rng = random.Random(8)
    docs = [cu.fuzz_doc_valid(rng) for _ in range(200)] + [MARKER] * 50
    data, off = pack(docs)
    res = scanner.lex_batch(data, off)
    full, total, rc = flat_index(scanner, reg, docs, doc_base=5, res=res)
    assert rc == 0 and total == len(full) >= 50
    part, total2, rc = flat_index(scanner, reg, docs, doc_base=5, cap=total - 1, res=res)
    assert rc == 0 and total2 == total and np.array_equal(part, full[:total - 1])
    none, total3, rc = flat_index(scanner, reg, docs, doc_base=5, cap=0, records=False, res=res)
    assert rc == 0 and total3 == total and len(none) == 0
    _e, total4, rc = flat_index(scanner, reg, [], res=scanner.lex_batch(np.zeros(0, np.uint8), np.zeros(1, np.uint64)))
    assert rc == 0 and total4 == 0


# ---------------------------------------------------------------------------------------------------------------------
# 4. the plain scan with d_bytes off 16-byte alignment
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_device_scan_unaligned_batch(scanner, oracle):
    """obm_lex_batch copies host batches into an aligned buffer; obm_lex_batch_device takes d_bytes as given.  Batches
    that start 1, 3, 8 and 15 bytes past a 16-byte boundary, well inside their allocation: modes 0-3 agree and match
    the oracle"""
    import torch
    import operator_builder_b200 as ob
    rng = random.Random(15)
    short = [ln * k for k in range(1, 40) for ln in (b"\n", b"#\n", b"+a:b\n", b"x\n+y:z=1\n", b"# +s:a=1,b\n")]
    corpora = [list(cu.TARGETED), list(cu.NON_ASCII), [cu.fuzz_doc(rng, max_len=300, non_ascii=k % 3 == 0) for k in range(1500)], short]
    for docs in corpora:
        data, off = pack(docs)
        want, want_off, _ = oracle.lex_batch_raw(data, off)
        scanner.set_mode(0)
        ref = scanner.lex_batch(data, off)
        cap = len(ref.tuples) + 64
        for skew in (1, 3, 8, 15):
            buf = torch.zeros(len(data) + 256, dtype=torch.uint8, device="cuda:0")
            assert buf.data_ptr() % 16 == 0
            buf[skew:skew + len(data)] = torch.from_numpy(data.copy()).to("cuda:0")
            d_off = to_dev(off)
            outs = []
            for mode in (0, 1, 2, 3):
                scanner.set_mode(mode)
                d_out = torch.full((cap,), -1, dtype=torch.int64, device="cuda:0")
                d_toff = torch.zeros(len(docs) + 1, dtype=torch.int64, device="cuda:0")
                d_status = torch.zeros(4, dtype=torch.int32, device="cuda:0")
                scanner.lex_batch_device(buf.data_ptr() + skew, d_off.data_ptr(), len(docs), len(data), d_out.data_ptr(), cap,
                                         d_toff.data_ptr(), d_status.data_ptr(), None, _stream())
                torch.cuda.synchronize()
                assert d_status.cpu().tolist()[0] == 0 and d_status.cpu().tolist()[3] == 0, (skew, mode)
                toff = d_toff.cpu().numpy().view(np.uint64)
                tup = d_out.cpu().numpy().view(np.uint64)[:int(toff[-1])]
                outs.append((tup, toff))
            scanner.set_mode(0)
            for tup, toff in outs:
                assert np.array_equal(tup, ref.tuples) and np.array_equal(toff, ref.doc_tuple_off), skew
            tup, toff = outs[0]
            for i, doc in enumerate(docs):
                got = ob.decode_doc_raw(doc, tup[int(toff[i]):int(toff[i + 1])])
                assert got == want[int(want_off[i]):int(want_off[i + 1])], (skew, i, doc[:100])
