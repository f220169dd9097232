"""Phase A of the fused warp kernel (obm_warp_core.h scan_range) walks the staged text a fixed number of bytes per lane
and step, and keeps its bitmaps in 32-byte words, newline prefixes per 64-byte word pair and W.naw per 1 KiB row.  These
host replays (the device source, run by 32 fibers per warp) put everything that geometry distinguishes -- line starts,
"//" pairs, document starts, bytes >= 0x80, carries across whole steps, range ends, paged units -- on both sides of
32-byte, 64-byte, 1 KiB and 2 KiB borders, and compare the tuple stream with the exact lexer's.  They hold for any step
width, so they also guard a change of it."""
import numpy as np
import pytest

from tests import hostsim

BUFB = 13312     # obm_warp.h: bytes staged per warp
MAXDOC = BUFB - 16
OWN_CAP = 256


def check(docs, skew=0, exact_docs=None):
    tup, toff, stats = hostsim.tile_batch(docs, skew, pipeline=2)
    for i, doc in enumerate(docs):
        want = hostsim.lex_doc(doc)
        got = tup[int(toff[i]):int(toff[i + 1])]
        if not np.array_equal(got, want):
            raise AssertionError(f"doc {i} (skew {skew}, {len(doc)} B) {doc[:120]!r}\n warp ={hostsim.fmt_tuples(got)[:40]}\n"
                                 f" exact={hostsim.fmt_tuples(want)[:40]}")
    assert int(toff[-1]) == len(tup)
    if exact_docs is not None:
        assert int(stats[2]) == exact_docs, stats  # documents the exact lexer took
    return stats


def filler(n, seed):
    """n bytes of manifest-like text: plain lines, comment lines, marker lines and "//" comments, with few enough
    owning lines (lines with a '#', '+' or "//") that a document of BUFB bytes stays below OWN_CAP"""
    rng = np.random.default_rng(seed)
    parts = [b"kind: Deployment\n", b"  replicas: 3 # +operator-builder:field:name=replicas,default=3,type=int\n",
             b"# plain comment\n", b"    image: nginx // +a:b=1\n", b"x\n", b"\n", b"  name: webstore # +op:f:n=x,t=string\n",
             b"+a:b:c='v',d\n", b"   #+x:y=2.5\n", b"labels: {a: b}\n"]
    parts += [b"  metadata:\n", b"    labels: {app: web, tier: front}\n", b"      - containerPort: 8080\n"] * 6
    out = bytearray()
    while True:
        part = parts[int(rng.integers(len(parts)))]
        if len(out) + len(part) > n:
            return bytes(out) + b"x" * (n - len(out))  # whole lines only: a cut marker line would take the exact lexer
        out += part


@pytest.mark.parametrize("skew", [1, 7, 15])
def test_ranges_ending_in_either_half_of_a_step(skew):
    """a unit's range [skew, skew + span) ends in the first or the second 1 KiB of a 2 KiB block, or on a border"""
    ends = [500, 1023, 1024, 1025, 1500, 2047, 2048, 2049, 3000, 3100, 4095, 4096, 4160, 5000, 6143, 6200, 8191, 9000, 10239, 11000, 12287]
    for k, end in enumerate(ends):
        n = end - skew
        check([filler(n, k)], skew, exact_docs=0)
        # the same span cut into documents
        text = filler(n, 100 + k)
        a = text.find(b"\n", n // 3) + 1 or n // 3   # cut at line ends: a cut marker line would take the exact lexer
        b = text.find(b"\n", a + n // 4) + 1 or a
        check([text[:a], text[a:b], text[b:]], skew, exact_docs=0)


def test_range_ending_next_to_the_end_of_the_buffer():
    """hi_pos within 64 bytes of BUFB: the end of the staged text and of the bitmaps"""
    for skew in (0, 1, 9, 15):
        for back in (1, 2, 15, 16, 17, 31, 32, 33, 63, 64):
            n = BUFB - back - skew
            if n > MAXDOC:
                continue
            check([filler(n, back)], skew, exact_docs=0)
            # two documents, both starting in the first tile (12 KiB)
            check([filler(12000, back), b"# +a:b=1\n" * 100 + filler(n - 12900, back)], skew, exact_docs=0)


BORDERS = [32, 64, 96, 992, 1024, 1056, 2016, 2048, 2080, 4096, 6144, 8192, 10240, 12256]


def at(skew, pos, body, tail=b"\n"):
    """a document whose byte `pos - skew` (buffer position pos) is the first byte of body"""
    return b"x" * (pos - skew) + body + tail


@pytest.mark.parametrize("skew", [0, 3, 15])
def test_events_on_both_sides_of_word_lane_and_step_borders(skew):
    for border in BORDERS:
        for d in (-2, -1, 0, 1):
            p = border + d
            if p - skew < 2:
                continue
            # a line start: the newline on one side, the line's first special on the other
            check([at(skew, p - 1, b"\n# +a:b:c=1,d\n")], skew, exact_docs=0)
            check([at(skew, p - 1, b"\n+a:b:c=1\n")], skew, exact_docs=0)
            check([at(skew, p - 1, b"\n//+a:b\n")], skew, exact_docs=0)
            # "//": the pair split by the border (and a lone '/' next to it)
            check([at(skew, p - 1, b"//+a:b=2 x\n")], skew, exact_docs=0)
            check([at(skew, p - 1, b"/x/ +a:b\n# c\n")], skew, exact_docs=0)
            check([at(skew, p - 1, b"/\n/+a:b\n")], skew, exact_docs=0)
            # a document start: the first document ends just before the border
            first = b"x" * (p - skew - 1) + b"/"
            check([first, b"/+a:b=3\n# c\n", b"#x\n"], skew, exact_docs=0)
            check([first[:-1] + b"\n", b"+a:b\n"], skew, exact_docs=0)
            check([first[:-1] + b"#", b"+a:b\n"], skew, exact_docs=0)
            # a byte >= 0x80 on either side: in a plain comment (line-parallel path) and on a marker line (exact lexer)
            check([at(skew, p - 1, "é # +a:b\n".encode()), b"# +c:d=1\n"], skew)
            check([at(skew, p - 2, b"# " + "é".encode() + b" c\n# +a:b=1\n"), b"+c:d\n"], skew, exact_docs=0)
            check([at(skew, p - 1, b"# +a:b=" + "é".encode())], skew, exact_docs=1)


def test_a_line_without_events_across_a_whole_step():
    """the first special of a line 2 KiB and more after its start: the carry runs through every lane of a step and across steps"""
    for skew in (0, 5, 15):
        for lead in (0, 1, 63, 64, 65, 2047, 2048, 2100):
            for length in (2048, 2112, 4096, 4200):
                doc = b"y" * lead + b"\n" + b"v" * length + b" # +a:b:c=1\n" + b"w" * length + b"//c\n"
                check([doc], skew, exact_docs=0)
                check([b"x" * lead + b"# c\n" + b"v" * length, b"z" * length + b"+a:b\n"], skew, exact_docs=0)


def test_paged_units():
    """more owning lines than the owner table in a unit of several documents: every document is scanned alone, with
    ranges that start and end anywhere inside a row"""
    for skew in (0, 6, 15):
        for lens in ((100, 120, 90), (255, 3, 200), (37, 250, 11, 64)):
            docs = [b"".join(b"# c%d\n" % (i % 7) for i in range(n)) for n in lens]
            check(docs, skew, exact_docs=0)
            docs = [b"".join((b"# +a:b:c=%d\n" % (i % 10)) if i % 3 == 0 else b"#x\n" for i in range(n)) for n in lens]
            check(docs, skew, exact_docs=0)


def test_more_owners_than_the_table():
    """one document with more than OWN_CAP owning lines cannot be paged: the exact lexer takes it"""
    for skew in (0, 11):
        for n in (OWN_CAP, OWN_CAP + 1, 700, 3000):
            doc = b"".join(b"#%d\n" % (i % 10) for i in range(n))
            check([doc], skew, exact_docs=0 if n <= OWN_CAP else 1)
            check([b"k: v\n", doc, b"+a:b\n"], skew)
