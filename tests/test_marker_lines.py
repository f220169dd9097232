"""The marker-line fast paths, edit by edit, against the oracle.

Every marker line of mode 0 goes through obmw::fast_line, k_warp_scan's phase C stepper (csrc/obm_warp.h): it emits the
tuples of a line inside the well-formed grammar  +scope:scope:arg=value,...  itself and hands anything else to the
generic lexer (FL_FALLBACK).  obm::Lexer::run_ascii (csrc/obm_core.h) holds its own copy of that grammar for modes 2 and
3, the ASCII chunk lexer of large documents and the generic hand-over itself.  The tests here walk the edge of that
grammar on purpose: about 60 templates, one production each, in 96 line contexts, and every one-byte replacement,
insertion and deletion and every truncation of them, at all 16 alignments, plus a seeded sample of two-edit lines.

- host, stepper alone (hostsim.fast_lines): every document whose marker lines all stay on the stepper must decode, with
  EOF, to the oracle's stream; its PackSink tuples must equal its DirectSink tuples unless the PackSink overflowed, and
  it overflows exactly when a line has more than LTS tuples or a len beyond ST_MAXLEN.  Every unedited template stays
  on the stepper; every template's edits both stay and fall back.
- host, the kernels' replays (warp, tile and pipeline): a subset, one line per document and many per document, and the
  staging limits (LTS, the 13-bit len of a staged tuple, the 8-bit distance of the first '+', MLCAP, the end of the
  document, bytes >= 0x80 next to a marker line) against the oracle; the warp replay's count of stepper and hand-over
  lines must equal the direct harness's.
- GPU: the same documents through modes 0-3 and edited lines joined into 20-60 KB documents (the chunk-parallel path).

The reference is always the C oracle; one fast path is never compared with the other.  Which edits fall back is not
pinned: a later stepper may accept more."""
import random
import time

import numpy as np
import pytest

from tests import hostsim

LTS = 24          # obm_warp.h: staged tuples per marker line
MLCAP = 32        # marker lines staged per unit
ST_MAXLEN = 8191  # largest len of a staged tuple (13 bits)
PD_GENERIC = 255  # orec plusd: '+' this far or farther after the line's first special -> the generic lexer
MAXDOC = 13296    # largest document the warp stages
N9 = b"9"

# one production each
TEMPLATES = [
    # scopes, flags, arguments
    b"+a:b", b"+a:b:c", b"+a:b:c:d", b"+operator-builder:field:name=replicas", b"+a:b=v", b"+a:flag", b"+a:b:flag",
    b"+a:b=1,flag,c=2", b"+a:b=1,flag", b"+a:b=1,f,g,h", b"+A.b-c/d:E_f=x", b"+a:b=v,c=w,d=x",
    # integers and floats
    b"+a:b=0", b"+a:b=-5", b"+a:b=007", b"+a:b=" + N9 * 17, b"+a:b=-" + N9 * 16, b"+a:b=" + N9 * 18, b"+a:b=-" + N9 * 17,
    b"+a:b=.5", b"+a:b=5.", b"+a:b=-.5", b"+a:b=123456789012345.5", b"+a:b=1.25,c=-3",
    # quoted strings: empty, holding delimiters, holding the other quote characters
    b"+a:b='x'", b"+a:b=\"x\"", b"+a:b=`x`", b"+a:b=''", b"+a:b=\"\"", b"+a:b=``", b"+a:b='a,b=c:d e+f'",
    b"+a:b=\"{x}[y](z);#//\"", b"+a:b=`:=, +;`", b"+a:b='q\"r`s'", b"+a:b=\"q'r`s\"", b"+a:b=`q'r\"s`", b"+a:b='x',c=\"y\"",
    # booleans
    b"+a:b=true", b"+a:b=false", b"+a:b=true,c=false", b"+a:b=false,c",
    # naked strings
    b"+a:b=x/y", b"+a:b=x.y", b"+a:b=v-1", b"+a:b=x_y", b"+a:b=x#y", b"+a:b=x;y", b"+a:b=x\ty", b"+a:b=x\ry", b"+a:b=v1.2-rc_3/x",
    b"+a:b=tru", b"+a:b=fals", b"+a:b=trux",
    # several markers on one line
    b"+a:b=1 +c:d", b"+a:b +c:d=x +e:f:g", b"+a:b='x' # +c:d=2", b"+a:b=v // +c:d",
]
# just past the stepper's 17-byte number limit: the generic lexer's unedited, the stepper's after a deletion
EDGE = {b"+a:b=" + N9 * 18, b"+a:b=-" + N9 * 17}
PREFIXES = [b"", b"#", b"# ", b"//", b"// ", b"key: v  # ", b"  - x # ", b"a/b: c # "]
SUFFIXES = [b"", b"\n", b"\r\n", b" tail", b" +x:y=1", b" # +c:d"]
FRONT = b"kind: Deployment\n"  # a plain line in front: the marker line is line 2 (a LINE tuple)
CONTEXTS = [(f, p, s) for f in (b"", FRONT) for p in PREFIXES for s in SUFFIXES]
# bytes of the host replays' single edits (the direct harness takes all of 0x00-0x7F)
SAMPLE = [0x00, 0x09, 0x0A, 0x0B, 0x0D, 0x20, 0x22, 0x23, 0x27, 0x2B, 0x2C, 0x2D, 0x2E, 0x2F, 0x30, 0x39, 0x3A, 0x3B, 0x3D,
          0x41, 0x5B, 0x5F, 0x60, 0x61, 0x65, 0x66, 0x74, 0x7B, 0x7F]


def pack(docs):
    data = np.frombuffer(b"".join(docs) + b"\0", dtype=np.uint8)[:-1]
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    return data, off


def in_context(body, ctx, tail=True):
    front, prefix, suffix = CONTEXTS[ctx]
    return front + prefix + body + (suffix if tail else b"")


def edited_lines(byte_set=range(128), seed=1, two_edits=60000):
    """-> (documents, template of each, edit kind of each, skew of each).  Kinds: 'base' (every template in every
    context), 'replace' / 'insert' (each byte of byte_set at each position), 'delete', 'truncate' (the document ends
    after the byte), 'two' (a seeded sample of two edits).  Skews are spread so that every position of every template
    is seen at all 16 alignments."""
    docs, tpl, kind, skew = [], [], [], []

    def add(d, t, k, s):
        docs.append(d); tpl.append(t); kind.append(k); skew.append(s & 15)

    for t, T in enumerate(TEMPLATES):
        for c in range(len(CONTEXTS)):
            add(in_context(T, c), t, "base", c + t)
        for i in range(len(T)):
            for b in byte_set:
                if b != T[i]:
                    add(in_context(T[:i] + bytes([b]) + T[i + 1:], (5 * i + b + t) % len(CONTEXTS)), t, "replace", i + b)
        for i in range(len(T) + 1):
            for b in byte_set:
                add(in_context(T[:i] + bytes([b]) + T[i:], (7 * i + b + 1 + t) % len(CONTEXTS)), t, "insert", i + b + 3)
        for i in range(len(T)):
            for s in range(16):
                add(in_context(T[:i] + T[i + 1:], (11 * i + s + t) % len(CONTEXTS)), t, "delete", s)
                add(in_context(T[:i + 1], (3 * i + s + t) % len(CONTEXTS), tail=False), t, "truncate", s)
    rng = random.Random(seed)
    bs = list(byte_set)
    for _ in range(two_edits):
        t = rng.randrange(len(TEMPLATES))
        T = bytearray(TEMPLATES[t])
        for _e in range(2):
            k, i = rng.randrange(3), rng.randrange(len(T) + 1)
            if k == 0 and i < len(T):
                T[i] = rng.choice(bs)
            elif k == 1 or len(T) == 0:
                T[i:i] = bytes([rng.choice(bs)])
            elif i < len(T):
                del T[i]
        add(in_context(bytes(T), rng.randrange(len(CONTEXTS))), t, "two", rng.randrange(16))
    return docs, np.array(tpl), np.array(kind), np.array(skew, dtype=np.uint8)


def first_difference(docs, got, got_off, want, want_off, what):
    for i in range(len(docs)):
        g, w = got[int(got_off[i]):int(got_off[i + 1])], want[int(want_off[i]):int(want_off[i + 1])]
        if g != w:
            import oracle
            raise AssertionError(f"{what}: document {i} {docs[i][:160]!r}\n got ={oracle.parse_stream(g)[:30]}\n"
                                 f" want={oracle.parse_stream(w)[:30]}")
    raise AssertionError(f"{what}: the streams differ in length only")


def oracle_streams(oracle, docs):
    data, off = pack(docs)
    stream, soff, _n = oracle.lex_batch_raw(data if len(data) else np.zeros(1, np.uint8), off)
    return stream, soff


def check_tuples(oracle, docs, tuples, toff, what, want=None):
    """every document's tuples (toff[d]:toff[d+1]) decode to the oracle's stream"""
    data, off = pack(docs)
    got, goff = hostsim.decode_batch(data, off, tuples, toff)
    want, woff = want or oracle_streams(oracle, docs)
    if got != want:
        first_difference(docs, got, goff, want, woff, what)


def check_direct(oracle, docs, skews, what):
    """the direct harness over docs -> info; asserts the stepper's contract on every document it takes"""
    data, off = pack(docs)
    info, direct, toff, staged, soff = hostsim.fast_lines(data, off, skews)
    took = info["res"] != hostsim.FLR_FALLBACK
    assert (info["ok"][took] == info["lines"][took]).all()
    # a document the stepper took, with EOF, decodes to the oracle's stream (handed-over documents have no tuples)
    sel = np.nonzero(took)[0]
    assert (np.diff(toff)[~took] == 0).all()
    sub = [docs[i] for i in sel]
    check_tuples(oracle, sub, direct, np.append(toff[sel], toff[-1]), what)
    # the PackSink overflows exactly when a line has more than LTS tuples or a len beyond ST_MAXLEN ...
    want_ovf = (info["max_tuples"] > LTS) | (info["max_len"] > ST_MAXLEN)
    bad = np.nonzero(took & (info["ovf"].astype(bool) != want_ovf))[0]
    assert len(bad) == 0, [(int(i), docs[i][:80], info[i]) for i in bad[:5]]
    # ... and holds the DirectSink's tuples when it does not
    same = took & ~want_ovf
    nd, ns = np.diff(toff).astype(np.int64), np.diff(soff).astype(np.int64)
    assert (nd[same] == ns[same]).all() and (ns[took & want_ovf] == 0).all()
    a, b = direct[np.repeat(same, nd)], staged[np.repeat(same, ns)]
    if not np.array_equal(a, b):
        d = int(np.repeat(np.nonzero(same)[0], nd[same])[np.nonzero(a != b)[0][0]])
        raise AssertionError(f"{what}: document {d} {docs[d][:80]!r}: staged tuples differ from the direct ones")
    return info


# ---------------------------------------------------------------------------------------------------------------------
# host: the stepper alone
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def edited():
    return edited_lines()


def test_templates_stay_on_the_stepper(oracle):
    """the floor a rewrite of phase C must keep: every unedited template, in every context, on the stepper.  A '\\r'
    before the newline is part of the last token for Go's lexer ('\\r' delimits nothing), so a number, bool or quoted
    value followed by "\\r\\n" is the generic lexer's; a name or naked string stays on the stepper"""
    docs, skews, where = [], [], []
    for t, T in enumerate(TEMPLATES):
        for c in range(len(CONTEXTS)):
            docs.append(in_context(T, c)); skews.append((c + t) & 15); where.append((t, c))
    info = check_direct(oracle, docs, np.array(skews, np.uint8), "templates")
    off_path = [(TEMPLATES[t], CONTEXTS[c]) for (t, c), r in zip(where, info["res"])
                if r != hostsim.FLR_OK and CONTEXTS[c][2] != b"\r\n" and TEMPLATES[t] not in EDGE]
    assert not off_path, off_path[:10]
    for T in EDGE:
        assert all(r == hostsim.FLR_FALLBACK for (t, _c), r in zip(where, info["res"]) if TEMPLATES[t] == T)
    assert (info["lines"] >= 1).all()


def test_every_edit_against_the_oracle(oracle, edited):
    docs, tpl, kind, skews = edited
    t0 = time.time()
    info = check_direct(oracle, docs, skews, "single and double edits")
    took = info["res"] == hostsim.FLR_OK
    lines, ok = int(info["lines"].sum()), int(info["ok"].sum())
    # both outcomes for every template: its edits cross the grammar's edge
    for t, T in enumerate(TEMPLATES):
        m = (tpl == t) & (kind != "base")
        assert took[m].any() and (info["res"][m] == hostsim.FLR_FALLBACK).any(), T
    # every single-edit position of every template at all 16 alignments
    single = np.isin(kind, ["replace", "insert", "delete", "truncate"])
    for t in range(len(TEMPLATES)):
        assert len(np.unique(skews[single & (tpl == t)])) == 16
    per_kind = {k: f"{took[kind == k].mean():.3f}" for k in ("base", "replace", "insert", "delete", "truncate", "two")}
    print(f"\nstepper harness: {len(docs)} documents, {lines} marker lines, {ok} on the stepper "
          f"({ok / lines:.3f}), {int(took.sum())} documents checked against the oracle, "
          f"{int((info['ovf'] != 0).sum())} PackSink overflows; acceptance by edit {per_kind}; {time.time() - t0:.1f} s")


# ---------------------------------------------------------------------------------------------------------------------
# host: the staging limits
# ---------------------------------------------------------------------------------------------------------------------
def staged_lines(n):
    """n marker lines of 9 tuples each (line >= 2): staged, far from LTS"""
    return b"".join(b"# +s:t=%d\n" % (k % 10) for k in range(n))


def line_of(ntuples):
    """a marker line (not the first line) of exactly ntuples tuples: LINE, Comment, 7 for '+a:b=1', 3 per ',c', 4 per ',d=1'"""
    for a in range(12):
        for b in range(12):
            if 9 + 3 * a + 4 * b == ntuples:
                return b"# +a:b=1" + b",c" * a + b",d=1" * b + b"\n"
    raise ValueError(ntuples)


def limit_docs():
    """documents of at most MAXDOC bytes at the stepper's staging limits, each beside ordinary staged lines"""
    docs = []
    head = b"k: v\n# +s:t=1\n"
    for n in (23, 24, 25):
        docs.append(head + line_of(n) + b"# +s:t=2\n")
        docs.append(head + staged_lines(MLCAP - 2) + line_of(n) + line_of(n) + b"# +s:t=2\n")  # 32nd and 33rd marker line
        docs.append(head + staged_lines(MLCAP - 1) + line_of(n) + b"k: v\n")
        docs.append(staged_lines(MLCAP - 1) + line_of(n))  # the 32nd marker line ends the document
    for n in range(ST_MAXLEN - 1, ST_MAXLEN + 3):
        docs.append(head + b"# +a:" + b"n" * n + b"=1\n" + b"# +s:t=2\n")        # a name
        docs.append(head + b"# +a:b=" + b"v" * n + b"\n" + b"# +s:t=2\n")        # a naked value
        docs.append(head + b"# +a:b='" + b"q" * n + b"'\n" + b"# +s:t=2\n")      # a quoted value
        docs.append(head + b"# +a:b=\"" + b"q" * (n - 2) + b"\",c\n")            # a quoted value n bytes with its quotes
        docs.append(head + b"# +a:b=`" + b"q" * (n - 2) + b"`")
    for line in (ST_MAXLEN - 1, ST_MAXLEN, ST_MAXLEN + 1, ST_MAXLEN + 2):
        docs.append(b"# +s:t=1\n" + b"\n" * (line - 2) + b"# +a:b=1,c\n" + b"# +s:t=2\n")  # the marker line is line `line`
        docs.append(b"# +s:t=1\n" + b"\n" * (line - 2) + b"x: 1 // +a:b")
    for k in (PD_GENERIC - 2, PD_GENERIC - 1, PD_GENERIC, PD_GENERIC + 1):
        for fill in (b"x", b" ", b"/", b"="):
            docs.append(head + b"# " + fill * (k - 2) + b"+a:b=1\n" + b"# +s:t=2\n")  # the first '+' k bytes after '#'
        docs.append(head + b"// " + b"y" * (k - 3) + b"+a:b +c:d=2\n")
        docs.append(head + b"k: v # " + b"z" * (k - 2) + b"+a:b\n")
    ends = [b"+a:b", b"+a:b=1", b"+a:b=-.5", b"+a:b='x'", b"+a:b=\"\"", b"+a:b=``", b"+a:b=true", b"+a:b=x;y", b"+a:b=1,c",
            b"+a:b c", b"+a:b +c:d", b"+a:b # +c:d=2", b"+a:b=1,c=2", b"+a:b:c=vvvvvvvvvvvvvvvvvvvvvvvvvvvvvv"]
    for j in range(16):  # a marker whose last token ends the document, the end at every offset of a 16-byte load
        for e in ends:
            docs.append(head + b"k" * j + b"\n# " + e)
    for e in ends[:6]:  # ... and in a document that fills the staged buffer
        body = b"# " + e
        filler = b"".join(b"key%d: value\n" % (k % 10) for k in range(1200))
        docs.append(filler[:MAXDOC - len(body) - 1] + b"\n" + body)
        assert len(docs[-1]) == MAXDOC
    for a, b in ((b"\xc3\xa9", b"\xc3\xa9"), (b"\xe2\x82\xac", b"\xf0\x9f\x98\x80"), (b"\xd0\xb6", b"")):
        for j in range(8):  # bytes >= 0x80 on the lines around a short marker line, in its 16-byte loads
            docs.append(head + b"k" * j + a + b"\n+a:b\n" + b + b": v\n")
            docs.append(head + b"k: " + a + b"\n# +a:b=1,c='" + b * 2 + b"x'\n" + b + b"\n")
            docs.append(b"k" * j + b"\n" + a + b"\n# +a:b=v" + b"\n" + b + b"\n")
    assert all(len(d) <= MAXDOC for d in docs)
    return docs


def test_staging_limits_in_the_stepper(oracle):
    docs = limit_docs()
    for s in range(16):
        info = check_direct(oracle, docs, np.full(len(docs), s, np.uint8), f"staging limits at skew {s}")
    assert (info["ovf"] != 0).sum() >= 10 and (info["max_tuples"] == LTS + 1).any() and (info["max_len"] == ST_MAXLEN + 1).any()


def replay_all(oracle, docs, what, skews=(0, 7), want_lines=None):
    """the warp replay (mode 0), the tile and pipeline replays (modes 2, 3) against the oracle.  want_lines: (stepper lines,
    hand-overs) the warp replay's phase C must count"""
    want = oracle_streams(oracle, docs)
    for skew in skews:
        f0, g0 = hostsim.warp_line_stats()
        tup, toff, _st, rep = hostsim.warp_batch(docs, skew)
        f1, g1 = hostsim.warp_line_stats()
        check_tuples(oracle, docs, tup, toff, f"{what}: warp replay at skew {skew}", want)
        if want_lines is not None:
            assert not rep["paged"].any()  # a paged unit scans its lines twice
            assert (f1 - f0, g1 - g0) == want_lines, (what, skew)
        for pipeline in (0, 1):
            tup, toff, _st = hostsim.tile_batch(docs, skew, pipeline=pipeline)
            check_tuples(oracle, docs, tup, toff, f"{what}: {'pipeline' if pipeline else 'tile'} replay at skew {skew}", want)
    return rep


def test_staging_limits_in_the_replays(oracle):
    # a plain 4 KB document after each: a tile starts few documents, so no unit has more owning lines than its table
    docs = [x for d in limit_docs() for x in (d, b"p: q\n" * 800)]
    data, off = pack(docs)
    info = hostsim.fast_lines(data, off, np.zeros(len(docs), np.uint8))[0]
    rep = replay_all(oracle, docs, "staging limits", skews=(0, 3, 9, 15),
                     want_lines=(int(info["ok"].sum()), int((info["lines"] - info["ok"]).sum())))
    assert rep["deferred"].any() and rep["needs_text"].any() and rep["long_line"].any()


# ---------------------------------------------------------------------------------------------------------------------
# host: through the kernels' replays
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sampled():
    docs, _tpl, _kind, _skews = edited_lines(SAMPLE, seed=2, two_edits=3000)
    return docs


def many_per_document(docs, per_doc=30):
    """lines joined per_doc to a document and padded with plain lines to 4 KiB: units of more than MLCAP marker lines
    (about four documents per tile), and not more owning lines than a unit's table"""
    out = []
    for k in range(0, len(docs), per_doc):
        body = b"\n".join(d.rstrip(b"\n") for d in docs[k:k + per_doc]) + b"\n"
        out.append(body + b"p: q\n" * max(0, (4096 - len(body)) // 5))
    return out


@pytest.mark.parametrize("layout", ["line_per_document", "lines_per_document"])
def test_edits_through_the_replays(oracle, sampled, layout):
    t0 = time.time()
    docs = sampled if layout == "line_per_document" else many_per_document(sampled)
    data, off = pack(docs)
    info = hostsim.fast_lines(data, off, np.zeros(len(docs), np.uint8))[0]
    ok, lines = int(info["ok"].sum()), int(info["lines"].sum())
    rep = replay_all(oracle, docs, layout, want_lines=(ok, lines - ok))
    if layout == "lines_per_document":
        assert hostsim.warp_units(off) > 100
    print(f"\n{layout}: {len(docs)} documents, {lines} marker lines ({ok} on the stepper, {lines - ok} handed over) through the "
          f"warp, tile and pipeline replays at 2 skews; {len(rep)} units, {int(rep['deferred'].sum())} deferred, "
          f"{int(rep['needs_text'].sum())} needs_text; {time.time() - t0:.1f} s")


def without_fatal(docs):
    """the documents without a fatal error (one would send a whole large document to the sequential lexer)"""
    return [d for d in docs if not ((hostsim.lex_doc(d) >> np.uint64(59)) >= 28).any()]


def large_documents(docs, seed=3):
    """edited lines joined into ASCII documents of 20 to 60 KB (the chunk-parallel path)"""
    rng = random.Random(seed)
    out, cur, size = [], [], rng.randint(20000, 60000)
    for d in docs:
        cur.append(d.rstrip(b"\n"))
        if sum(len(x) + 1 for x in cur) >= size:
            out.append(b"\n".join(cur) + b"\n")
            cur, size = [], rng.randint(20000, 60000)
    return out


def test_large_documents_of_edited_lines(oracle, sampled):
    docs = large_documents(without_fatal(sampled)) + large_documents(sampled[::5])
    want, woff = oracle_streams(oracle, docs)
    chained = 0
    for i, d in enumerate(docs):
        tup, used = hostsim.large_doc(d)
        chained += used
        got = hostsim.decode(d, tup)
        assert got == want[int(woff[i]):int(woff[i + 1])], i
    assert chained >= len(docs) // 2, (chained, len(docs))
    print(f"\n{len(docs)} documents of 20-60 KB, {chained} through chains that validated")


# ---------------------------------------------------------------------------------------------------------------------
# GPU: modes 0-3
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scanner():
    import operator_builder_b200 as ob
    sc = ob.Scanner(0)
    yield sc
    sc.set_mode(0)
    sc.close()


def device_modes(scanner, oracle, docs, what):
    data, off = pack(docs)
    want = oracle_streams(oracle, docs)
    first = None
    for mode in (0, 1, 2, 3):
        scanner.set_mode(mode)
        res = scanner.lex_batch(data, off)
        check_tuples(oracle, docs, res.tuples, res.doc_tuple_off, f"{what}: mode {mode}", want)
        if first is None:
            first = res
        else:
            assert np.array_equal(res.doc_tuple_off, first.doc_tuple_off), (what, mode)
            assert np.array_equal(res.tuples, first.tuples), (what, mode)
    scanner.set_mode(0)
    print(f"\n{what}: {len(docs)} documents, {len(data)} bytes, {len(first.tuples)} tuples, modes 0-3 equal to the oracle")


@pytest.mark.gpu
def test_edits_on_device(scanner, oracle, edited):
    docs = edited[0]
    device_modes(scanner, oracle, docs, "single and double edits")
    device_modes(scanner, oracle, many_per_document(docs[::7]), "edits, many lines per document")


@pytest.mark.gpu
def test_staging_limits_on_device(scanner, oracle):
    device_modes(scanner, oracle, limit_docs(), "staging limits")


@pytest.mark.gpu
def test_large_documents_on_device(scanner, oracle, edited):
    docs = edited[0][::2]
    device_modes(scanner, oracle, large_documents(without_fatal(docs)) + large_documents(docs[::5]), "documents of 20-60 KB")
