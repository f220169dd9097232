"""obm_lex_collection_batch_device: Manifest.LoadContent's collection rewrite (manifests/manifest.go:89-95) fused into the
warp scan.  Its outputs must equal the composition obm_rewrite_collection_markers_device -> obm_lex_batch_device bit for
bit, and the lexemes must equal the oracle's over the documents rewritten by Python's bytes.replace (Go's ReplaceAll).

CPU: the device source of the collection variant (compute_unit<true> + write_text) replayed on the host by 32 fibers per
warp (tests/hostsim/collection.cpp), against the Python rewrite followed by the host lexer.  GPU: the library itself."""
import random

import numpy as np
import pytest

from tests import corpus_util as cu
from tests import hostsim
from tests.hostsim import collection as hs_collection

P1, P2 = b"+operator-builder:collection:field", b"collectionField"
TILE, ROW, MAXDOC = 12288, 1024, 13296  # obm_warp.h: a unit's tile, phase A's row, the largest document a unit holds


def rewrite(doc: bytes) -> bytes:
    return doc.replace(P1, b"+operator-builder:field").replace(P2, b"field")


# ---- corpora ------------------------------------------------------------------------------------------------------
def corpus_fixtures():
    return [d for _p, d in cu.fixtures()]


def corpus_flavour1(n=48):
    import operator_builder_b200 as ob
    data, off = ob.generate_corpus_host(n, 4096, flavour=1)
    raw = data.tobytes()
    return [raw[int(off[i]):int(off[i + 1])] for i in range(n)]


def corpus_patterns():
    """the rewrite's pattern edge cases: overlapping spellings, truncated patterns, patterns cut by a document border,
    dense patterns, empty documents"""
    rng = random.Random(7)
    docs = [b"collectionFcollectionField", P2, P1, P1[:-1], P2[:-1], P2[:10], b"Field", b"+operator-builder:collection:", b"field",
            P2[:7], P2[7:], P1[:20], P1[20:] + P2, b"", b"", b"xcollectionFieldcollectionField" + P1 + b"x",
            b"+operator-builder:+operator-builder:collection:fieldcollectionFieldcollectionField",
            b"++operator-builder:collection:field:name=collectionField\n", b"+operator-builder:collection:collectionField",
            P2 * 300, (P1 + b"\n") * 100, (b"# " + P1 + b":name=a" + P2 + b",type=string\n") * 40]
    for _ in range(150):
        parts = [rng.choice([P1, P2, P1[:rng.randint(0, 34)], P2[:rng.randint(0, 15)], b"\n", b"# ", b"x" * rng.randint(0, 90), b"F", b"+",
                             b":name=a,type=string", b"c"]) for _ in range(rng.randint(0, 8))]
        docs.append(b"".join(parts))
    return docs


def corpus_shifts():
    """a pattern at every shift across 1 KiB row borders and 16-byte boundaries: one 12 KiB document per unit, patterns
    ending around row borders inside it and around its own end (the next unit's border: the pattern is then cut)"""
    docs = []
    for s in range(0, 40):
        d = bytearray(b"a" * TILE)
        for k, pat in enumerate((P1, P2, P1, P2)):
            at = ROW * (2 + 3 * k) - s
            d[at:at + len(pat)] = pat
        d[TILE - 60 - s:TILE - 45 - s] = P2
        d[TILE - 10:] = P1[:10]  # cut by the document's end
        docs.append(bytes(d))
        docs.append(P1[10:] + b"\n")  # ... and continued in the next document: no match
    return docs


def corpus_units():
    """units of 31 small documents, paged units (more owning lines than a unit's owner table, 16-byte lines carrying
    patterns), documents for the exact lexer (text beyond ASCII on a marker line with a pattern, a back-tick value over
    several lines, a fatal error)"""
    docs = [b"# " + P1 + b":name=d%d,type=int\nk: v # %s\n" % (i, P2) for i in range(70)]
    docs += [b"#collectionField\n" * 200, b"# c\n" * 100 + b"#" + P1 + b"\n", b"#collectionField\n" * 150 + b"x: y\n"] * 2
    docs += ["# +operator-builder:collection:field:name=été,type=string\n".encode(),
             "café: 1 # plain\n# +operator-builder:collection:field:name=a\n".encode(),
             b"# +operator-builder:collection:field:name=`multi\n  # line collectionField`,type=string\n",
             b"+a:b=1e309\n# " + P1 + b":name=x\n", b"# +operator-builder:collection:field:name=\"unterminated\nk: v\n", b""]
    return docs


def corpus_large():
    """documents above MAXDOC: rewritten on the large path; one shrinks below MAXDOC, two are adjacent"""
    line = b"  - item  # " + P1 + b":name=a.b,type=int,default=3\n"
    big = (line + b"key: value\n") * 400
    shrink = (b"# " + P1 + b"\n") * (MAXDOC // 36 + 2)
    assert len(shrink) > MAXDOC and len(rewrite(shrink)) < MAXDOC
    return [b"k: v # " + P1 + b":name=x\n", big, shrink, b"", big[:20000], b"collectionField\n", P2 * 1000, b"tail " + P1 + b"\n"]


CPU_CORPORA = {"fixtures": corpus_fixtures, "flavour1": corpus_flavour1, "patterns": corpus_patterns, "shifts": corpus_shifts,
               "units": corpus_units, "large": corpus_large}


# ---- CPU: the host replay of the collection variant ----------------------------------------------------------------
def check_host(docs, skew=0):
    out_bytes, out_off, tuples, toff, _stats = hs_collection.collection_batch(docs, skew)
    want = [rewrite(d) for d in docs]
    end = int(out_off[-1])
    assert end == sum(len(w) for w in want)
    assert out_bytes[end:end + 16] == b"\xee" * 16, "bytes written past the rewritten batch"
    for i, w in enumerate(want):
        assert out_bytes[int(out_off[i]):int(out_off[i + 1])] == w, (i, docs[i][:80])
        got = tuples[int(toff[i]):int(toff[i + 1])]
        exp = hostsim.lex_doc(w)
        assert len(got) == len(exp) and np.array_equal(got, exp), (i, docs[i][:80], hostsim.fmt_tuples(got)[:20], hostsim.fmt_tuples(exp)[:20])
    assert int(toff[-1]) == len(tuples)


@pytest.mark.parametrize("name", sorted(CPU_CORPORA))
def test_host_collection_variant(name):
    docs = CPU_CORPORA[name]()
    assert docs
    for skew in (0, 5):
        check_host(docs, skew)


def test_host_collection_variant_rewrites_something():
    docs = corpus_flavour1(8)
    assert sum(rewrite(d) != d for d in docs) == 8  # the collection spelling: every document has patterns


def test_host_stale_shared_memory_between_units():
    """a batch of long units, then short ones: what the long ones left in the warp's buffer must not matter (the replay
    keeps its shared memory across calls, like a persistent warp across units)"""
    long_docs = [(b"# " + P1 + b":name=a\n" + b"+" * 200 + b"\n") * 50]
    check_host(long_docs)
    check_host([b"k: v\n", P2[:12], b"# +x:y=1\n", b"collectionFiel", b"", b"+operator-builder:collection:fiel"])
    check_host(long_docs + [b"# " + P2] * 3)


def test_host_empty_batch():
    out_bytes, out_off, tuples, toff, _ = hs_collection.collection_batch([])
    assert len(tuples) == 0 and int(out_off[0]) == 0 and int(toff[0]) == 0


# ---- GPU: the library -------------------------------------------------------------------------------------------------
def _dev(docs, byte_shift=0):
    import torch
    data = np.frombuffer(b"".join(docs) + b"\0", dtype=np.uint8)[:-1].copy()
    off = np.zeros(len(docs) + 1, dtype=np.int64)
    if docs:
        off[1:] = np.cumsum([len(d) for d in docs])
    raw = torch.zeros(len(data) + 64 + byte_shift, dtype=torch.uint8, device="cuda:0")
    raw[byte_shift:byte_shift + len(data)] = torch.from_numpy(data).to("cuda:0")
    return raw[byte_shift:], torch.from_numpy(off).to("cuda:0"), off


def _outputs(n_bytes, ndocs, cap):
    import torch
    return dict(bytes=torch.full((n_bytes + 64,), 0xEE, dtype=torch.uint8, device="cuda:0"),
                doc_off=torch.full((ndocs + 1,), -1, dtype=torch.int64, device="cuda:0"),
                out=torch.full((cap + 16,), -1, dtype=torch.int64, device="cuda:0"),
                toff=torch.full((ndocs + 1,), -1, dtype=torch.int64, device="cuda:0"),
                status=torch.full((4,), -1, dtype=torch.int32, device="cuda:0"),
                counts=torch.full((2,), -1, dtype=torch.int64, device="cuda:0"))


def _fused(sc, d_bytes, d_off, ndocs, total, o, cap, mode=0):
    import torch
    old = sc.set_mode(mode)
    try:
        sc.lex_collection_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, total, o["bytes"].data_ptr(), total, o["doc_off"].data_ptr(),
                                       o["out"].data_ptr(), cap, o["toff"].data_ptr(), o["status"].data_ptr(), o["counts"].data_ptr(),
                                       torch.cuda.current_stream().cuda_stream)
    finally:
        sc.set_mode(old)
    torch.cuda.synchronize()


def _composition(sc, d_bytes, d_off, ndocs, total, o, cap):
    import torch
    from operator_builder_b200 import _native
    st = torch.cuda.current_stream().cuda_stream
    rc = _native.lib().obm_rewrite_collection_markers_device(sc.handle, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, o["bytes"].data_ptr(), total,
                                                             o["doc_off"].data_ptr(), st)
    assert rc == 0
    torch.cuda.synchronize()
    rewritten = int(o["doc_off"][ndocs].item()) if ndocs else 0
    sc.lex_batch_device(o["bytes"].data_ptr(), o["doc_off"].data_ptr(), ndocs, rewritten, o["out"].data_ptr(), cap, o["toff"].data_ptr(),
                        o["status"].data_ptr(), o["counts"].data_ptr(), st)
    torch.cuda.synchronize()


def _same(a, b, status_words=(0, 1, 2, 3)):
    import torch
    for k in ("bytes", "doc_off", "out", "toff", "counts"):
        assert torch.equal(a[k], b[k]), k
    for w in status_words:
        assert int(a["status"][w].item()) == int(b["status"][w].item()), w


def compare_on_device(sc, oracle, docs, byte_shift=0, cap=None, with_oracle=True):
    """fused (mode 0) == composition in mode 0 == the fused call in mode 1 (which runs the composition with the exact
    lexer); then the lexemes against the oracle over the Python-rewritten documents"""
    import operator_builder_b200 as ob
    d_bytes, d_off, off = _dev(docs, byte_shift)
    ndocs, total = len(docs), int(off[-1])
    cap = cap if cap is not None else 2 * total + 2 * ndocs + 16
    fused = _outputs(total, ndocs, cap)
    _fused(sc, d_bytes, d_off, ndocs, total, fused, cap)
    comp = _outputs(total, ndocs, cap)
    _composition(sc, d_bytes, d_off, ndocs, total, comp, cap)
    # status[1] counts the documents the exact lexer took: a document above MAXDOC takes the large path in the fused call
    # even when its rewritten text is shorter, while the composition lexes the rewritten text line-parallel
    shrinks = any(len(d) > MAXDOC >= len(rewrite(d)) for d in docs)
    _same(fused, comp, status_words=(0, 2, 3) if shrinks else (0, 1, 2, 3))
    exact = _outputs(total, ndocs, cap)
    _fused(sc, d_bytes, d_off, ndocs, total, exact, cap, mode=1)
    _same(fused, exact, status_words=(0, 2))  # status[1] counts the documents the exact lexer took: all of them in mode 1
    want = [rewrite(d) for d in docs]
    noff = fused["doc_off"].cpu().numpy()
    out_bytes = fused["bytes"].cpu().numpy().tobytes()
    assert int(noff[-1]) == sum(len(w) for w in want)
    assert out_bytes[int(noff[-1]):] == b"\xee" * (len(out_bytes) - int(noff[-1])), "bytes written past out_doc_off[ndocs]"
    for i, w in enumerate(want):
        assert out_bytes[int(noff[i]):int(noff[i + 1])] == w, (i, docs[i][:80])
    if with_oracle and int(fused["status"][0].item()) == 0:
        tuples = fused["out"].cpu().numpy().view(np.uint64)
        toff = fused["toff"].cpu().numpy().view(np.uint64)
        wdata = np.frombuffer(b"".join(want) + b"\0", dtype=np.uint8)[:-1]
        woff = np.zeros(ndocs + 1, dtype=np.uint64)
        woff[1:] = np.cumsum([len(w) for w in want]) if want else []
        want_stream, want_off, _n = oracle.lex_batch_raw(wdata if len(wdata) else np.zeros(1, np.uint8), woff)
        for i, w in enumerate(want):
            got = ob.decode_doc_raw(w, tuples[int(toff[i]):int(toff[i + 1])])
            assert got == want_stream[int(want_off[i]):int(want_off[i + 1])], (i, docs[i][:80])
    return fused


@pytest.fixture(scope="module")
def scanner():
    import operator_builder_b200 as ob
    sc = ob.Scanner(0)
    yield sc
    sc.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CPU_CORPORA))
def test_device_fused_equals_composition(scanner, oracle, name):
    compare_on_device(scanner, oracle, CPU_CORPORA[name]())


@pytest.mark.gpu
def test_device_fused_10k_flavour1(scanner, oracle):
    compare_on_device(scanner, oracle, corpus_flavour1(10000))


@pytest.mark.gpu
def test_device_large_documents(scanner, oracle):
    docs = corpus_large()
    rng = random.Random(3)
    docs += [b"".join(rng.choice([P1 + b"\n", P2, b"k: v\n", b"# " + P1 + b":name=a\n", b"x" * 200]) for _ in range(rng.randint(600, 3000)))
             for _ in range(6)]
    docs += [docs[1], docs[1], b"", docs[2]]  # adjacent large documents
    compare_on_device(scanner, oracle, docs)


@pytest.mark.gpu
def test_device_unaligned_input(scanner, oracle):
    compare_on_device(scanner, oracle, corpus_patterns() + corpus_large(), byte_shift=3)


@pytest.mark.gpu
def test_device_no_documents(scanner, oracle):
    compare_on_device(scanner, oracle, [])
    compare_on_device(scanner, oracle, [b"", b""])


@pytest.mark.gpu
def test_device_tuple_capacity(scanner, oracle):
    """out_cap too small: status[0] as for obm_lex_batch_device, nothing written past out_cap; the bytes are complete"""
    fused = compare_on_device(scanner, oracle, corpus_flavour1(200), cap=1000, with_oracle=False)
    assert int(fused["status"][0].item()) == 1
    assert bool((fused["out"][1000:] == -1).all())


@pytest.mark.gpu
def test_device_bad_arguments(scanner):
    import torch
    from operator_builder_b200 import _native
    docs = corpus_flavour1(4)
    d_bytes, d_off, off = _dev(docs)
    total = int(off[-1])
    o = _outputs(total, 4, 4096)
    L = _native.lib()
    st = torch.cuda.current_stream().cuda_stream
    args = lambda ob_, cap_: (scanner.handle, d_bytes.data_ptr(), d_off.data_ptr(), 4, total, ob_, cap_, o["doc_off"].data_ptr(),
                              o["out"].data_ptr(), 4096, o["toff"].data_ptr(), None, None, st)
    assert L.obm_lex_collection_batch_device(*args(o["bytes"].data_ptr(), total - 1)) == _native.OBM_E_ARG  # out_bytes_cap < total_bytes
    assert L.obm_lex_collection_batch_device(*args(o["bytes"].data_ptr() + 1, total)) == _native.OBM_E_ARG  # not 16-byte aligned
    assert L.obm_lex_collection_batch_device(*args(d_bytes.data_ptr(), total)) == _native.OBM_E_ARG  # overlaps the input
    torch.cuda.synchronize()
    assert bool((o["bytes"] == 0xEE).all())


@pytest.mark.gpu
def test_device_full_size_c3(scanner, oracle):
    """C3 at full size (1,048,576 x 4 KiB, flavour 1, generated on the device): fused == composition on the device, and the
    per-document hash of the fused stream over the rewritten bytes == the oracle's over the same bytes"""
    import os
    import torch
    from operator_builder_b200 import _native
    ndocs, doc_bytes = 1048576, 4096
    total = ndocs * doc_bytes
    free, _ = torch.cuda.mem_get_info()
    if free < 6 * total + (4 << 30):
        pytest.skip("not enough free HBM for C3 at full size")
    st = torch.cuda.current_stream().cuda_stream
    d_bytes = torch.empty(total + 64, dtype=torch.uint8, device="cuda:0")
    d_off = torch.empty(ndocs + 1, dtype=torch.int64, device="cuda:0")
    scanner.generate_corpus_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, doc_bytes, 0, 1, st)
    cap = total // 16
    fused = _outputs(total, ndocs, cap)
    _fused(scanner, d_bytes, d_off, ndocs, total, fused, cap)
    comp = _outputs(total, ndocs, cap)
    _composition(scanner, d_bytes, d_off, ndocs, total, comp, cap)
    _same(fused, comp)
    del comp
    torch.cuda.empty_cache()
    assert int(fused["status"][0].item()) == 0 and int(fused["counts"][0].item()) == 8 * ndocs
    d_hash = torch.zeros(ndocs, dtype=torch.int64, device="cuda:0")
    d_nhost = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    rc = _native.lib().obm_hash_batch_device(scanner.handle, fused["bytes"].data_ptr(), fused["doc_off"].data_ptr(), ndocs, fused["out"].data_ptr(),
                                             fused["toff"].data_ptr(), d_hash.data_ptr(), d_nhost.data_ptr(), st)
    assert rc == 0
    torch.cuda.synchronize()
    assert int(d_nhost.item()) == 0
    got = d_hash.cpu().numpy().view(np.uint64)
    noff = fused["doc_off"].cpu().numpy().astype(np.uint64)
    host = fused["bytes"][:int(noff[-1])].cpu().numpy()
    assert int(noff[-1]) < total  # the collection spelling shrinks
    del fused, d_bytes
    torch.cuda.empty_cache()
    threads = max(1, len(os.sched_getaffinity(0)))
    _n_lex, n_mark, _h, want = oracle.scan_batch(host, noff, threads, want_doc_hash=True)
    assert n_mark == 8 * ndocs
    bad = np.nonzero(got != want)[0]
    assert len(bad) == 0, (len(bad), bad[:10])
