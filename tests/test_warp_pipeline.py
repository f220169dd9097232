"""k_warp_scan's software pipeline over the units a warp takes one after another (obm_warp.cuh): after unit i is scanned
and has published its count, the warp stages unit i + 1's text over unit i's and loads its document offsets (when
prestage_next allows it), writes unit i - 1 from W.fin, and only then assembles unit i into W.fin or writes it directly.
Only a warp's second and later units go through that: the text under a direct write (more than FIN_CAP tuples,
long_line) is already the next unit's, and a unit whose write lexes its text again (needs_text: exact documents,
marker lines that are not staged, paged units) must not be staged over.

The batches here are made of tile-aligned segments of named unit classes, laid out in runs and interleaved so that
every ordered pair of classes meets.  On the host, the replay (hostsim.warp_batch) runs the pipeline in the kernel's
order, lands each bulk copy at once over poisoned text, and reports how every unit went; its tuples must be the exact
lexer's, and the report must show the hand-overs above.  On the GPU, the same classes at a size that gives every
resident warp at least 8 units run through all four scan organisations and are checked against the oracle."""
import os
import random
import time

import numpy as np
import pytest

from tests import corpus_util as cu
from tests import hostsim

TILE = 12288      # obm_warp.h: a unit = the documents that start in one TILE-byte range of the batch
BUFB = 13312      # bytes staged per warp
MAXDOC = BUFB - 16  # larger documents take the chunk-parallel exact path (an `extra` unit)
DMAX = 31         # documents per unit
FIN_CAP = 704     # tuples of a unit whose write is deferred
ST_MAXLEN = 8191  # line numbers the packed tuple holds (more: long_line)
WPC = 10          # k_warp_scan: warps per CTA, one CTA per SM

YAML = [b"kind: Deployment\n", b"metadata:\n", b"  name: webstore\n", b"    labels: {app: web, tier: front}\n", b"spec:\n",
        b"      - containerPort: 8080\n", b"  replicas: 3\n", b"    image: nginx:1.17\n", b"  data: [1, 2]\n", b"\n"]
MARKED = [b"  replicas: 3 # +operator-builder:field:name=replicas,default=3,type=int\n", b"    image: nginx // +a:b=1\n",
          b"  name: webstore # +op:f:n=x,t=string\n", b"  # +x:y:z='v',w\n", b"# +a:b=\"q q\",c=1.5,d=true\n"]
COMMENTS = [b"# plain comment\n", b"  # see https://x/y\n", b"// go comment\n"]


def manifest(rng, n):
    """exactly n bytes (n > 0) of whole manifest lines, a marker line (at most 24 tuples) every ~30 lines: about 17 per
    tile, far from the 32 staged ones and from FIN_CAP"""
    out = bytearray()
    while True:
        k = rng.random()
        part = rng.choice(MARKED) if k < 0.035 else rng.choice(COMMENTS) if k < 0.07 else rng.choice(YAML)
        if len(out) + len(part) > n - 1:
            return bytes(out) + b"x" * (n - 1 - len(out)) + b"\n"
        out += part


def plain(rng, n):
    """exactly n bytes (n > 0) of lines without a '#', '+' or "//": no owning line, no tuple but EOF"""
    out = bytearray()
    while len(out) < n - 1:
        out += b"  key%d: value %d\n" % (rng.randrange(1000), rng.randrange(10 ** rng.randint(1, 9)))
    return bytes(out[:n - 1]) + b"\n"


def fill(rng, docs, total):
    """docs plus one manifest document that brings their length to `total` (none when it already is)"""
    n = total - sum(len(d) for d in docs)
    assert n >= 0
    return docs + [manifest(rng, n)] if n else docs


def marker_line(rng):
    """a marker line the stepper stages: 9 to 21 tuples"""
    args = ",".join("%s=%d" % (c, rng.randrange(100)) for c in "bcde"[:rng.randint(1, 4)])
    return b"# +a:%s\n" % args.encode()


# ---- the unit classes: f(rng, large_sizes) -> documents whose lengths add up to a multiple of TILE ----------------------
def c_manifest_4k(rng, _ls):
    return [manifest(rng, 4096) for _ in range(3)]


def c_over_fin_cap(rng, _ls):
    """32 staged marker lines and 60 plain comment lines in one unit: 21 * 32 + 2 * 60 tuples > FIN_CAP, all staged"""
    docs = []
    for _ in range(2):
        lines = [b"# +a:b=%d,c=%d,d=%d,e=%d\n" % tuple(rng.randrange(100) for _ in range(4)) for _ in range(16)]
        lines += [b"# note %d\n" % rng.randrange(10) for _ in range(30)]
        rng.shuffle(lines)
        body = b"k: v\n" + b"".join(lines)
        docs.append(body + plain(rng, 6144 - len(body)))
    return docs


def c_many_marker_lines(rng, _ls):
    """more than 32 marker lines: the ones after the 32nd are not staged (needs_text)"""
    body = b"".join(marker_line(rng) for _ in range(rng.randint(33, 80)))
    return fill(rng, [body + manifest(rng, 4096)], TILE)


def c_paged(rng, _ls):
    """short comment lines: more owning lines than the owner table in a unit of several documents"""
    docs = []
    for _ in range(6):
        body = b"".join((marker_line(rng) if k % 9 == 0 else b"#c\n") for k in range(rng.randint(60, 120)))
        docs.append(body + manifest(rng, 2048 - len(body)))
    return docs


def c_non_ascii(rng, _ls):
    """a marker line with bytes >= 0x80: the exact lexer inside the warp"""
    bad = rng.choice(["# +a:b=café\n", "# +été:nom=x\n", "  k: v # +a:b='€',c\n"]).encode()
    doc = manifest(rng, 2000) + bad
    return fill(rng, [manifest(rng, 4096), doc + manifest(rng, 4096 - len(doc))], TILE)


def c_long_line(rng, _ls):
    """comments after more than ST_MAXLEN empty lines: long_line, the unit cannot take the deferred write.  (A marker line
    there would not be staged, as its LINE tuple does not fit the packed form: needs_text.)"""
    doc = manifest(rng, 1000) + b"\n" * (ST_MAXLEN + rng.randint(1, 300)) + b"# c\n// d\n"
    return fill(rng, [doc], TILE)


def c_doc_maxdoc(rng, _ls):
    """a document of MAXDOC bytes: the largest that is staged"""
    return fill(rng, [manifest(rng, MAXDOC)], 2 * TILE)


def c_doc_maxdoc_plus1(rng, _ls):
    """a document of MAXDOC + 1 bytes: the smallest that takes the large path"""
    return fill(rng, [manifest(rng, MAXDOC + 1)], 2 * TILE)


def c_large(rng, large_sizes):
    """a large document after none to three small ones in its tile (none: an nd = 0 unit), then the rest of its tiles"""
    small = [manifest(rng, rng.randint(200, 1500)) for _ in range(rng.choice([0, 0, 1, 3]))]
    n = rng.choice(large_sizes)
    docs = small + [manifest(rng, n)]
    total = sum(len(d) for d in docs)
    return fill(rng, docs, -(-total // TILE) * TILE)


def c_docs_31(rng, _ls):
    """exactly DMAX documents in one tile"""
    return [manifest(rng, 396) for _ in range(30)] + [manifest(rng, TILE - 30 * 396)]


def c_empty_docs(rng, _ls):
    """empty documents: a unit of 31 of them (span 0), then more among non-empty ones"""
    docs = [b""] * 33 + [manifest(rng, 4096)]
    for _ in range(2):
        docs += [b"", manifest(rng, 4096)]  # none at the end: it would start the next segment's tile
    return docs


def c_fuzz(rng, _ls):
    """cu.fuzz_doc and cu.fuzz_doc_valid documents (warnings, fatal errors, bytes >= 0x80, odd line shapes)"""
    docs, total = [], 0
    while True:
        k = rng.random()
        d = cu.fuzz_doc(rng, max_len=600, non_ascii=k < 0.3) if k < 0.6 else cu.fuzz_doc_valid(rng, max_lines=rng.choice([2, 8, 30]))
        if total + len(d) > TILE - 64:
            return fill(rng, docs, TILE)
        docs.append(d)
        total += len(d)


CLASSES = {f.__name__[2:]: f for f in (c_manifest_4k, c_over_fin_cap, c_many_marker_lines, c_paged, c_non_ascii, c_long_line,
                                       c_doc_maxdoc, c_doc_maxdoc_plus1, c_large, c_docs_31, c_empty_docs, c_fuzz)}


def pool(seed, per_class, large_sizes):
    """per_class instances of every class -> {name: [documents of one segment, ...]}"""
    rng = random.Random(seed)
    out = {}
    for name, f in CLASSES.items():
        out[name] = []
        for _ in range(per_class):
            docs = f(rng, large_sizes)
            assert sum(len(d) for d in docs) % TILE == 0, name
            out[name].append(docs)
    return out


def runs(rng, names, n_runs):
    """runs of 1 to 12 segments of one class, every class in turn"""
    order = []
    while len(order) < n_runs:
        order += rng.sample(names, len(names))
    return [name for name in order[:n_runs] for _ in range(rng.randint(1, 12))]


def pairs(names):
    """every ordered pair of classes back to back"""
    return [x for a in names for b in names for x in (a, b)]


def assemble(rng, segs, layout):
    """class names -> (documents, the class of each document's segment)"""
    docs, cls = [], []
    for name in layout:
        seg = rng.choice(segs[name])
        docs += seg
        cls += [name] * len(seg)
    return docs, cls


def hand_overs(rep):
    """counts of the pipeline's hand-overs between consecutive units of a report"""
    a, b = rep[:-1], rep[1:]
    direct = (a["needs_text"] == 0) & (a["deferred"] == 0)
    return {
        "units": len(rep),
        "prestaged": int(rep["prestaged"].sum()),
        "deferred": int(rep["deferred"].sum()),
        "needs_text": int(rep["needs_text"].sum()),
        "paged": int(rep["paged"].sum()),
        "over_fin": int(rep["over_fin"].sum()),
        "long_line": int(rep["long_line"].sum()),
        "extra": int(rep["extra"].sum()),
        "prestaged_after_deferred": int(((a["deferred"] == 1) & (b["prestaged"] == 1)).sum()),
        "prestaged_after_fin_cap_write": int((direct & (a["over_fin"] == 1) & (b["prestaged"] == 1)).sum()),
        "prestaged_after_long_line_write": int((direct & (a["long_line"] == 1) & (b["prestaged"] == 1)).sum()),
        "staged_after_needs_text": int(((a["needs_text"] == 1) & (a["paged"] == 0) & (b["nd"] > 0) & (b["prestaged"] == 0)).sum()),
        "staged_after_paged": int(((a["paged"] == 1) & (b["nd"] > 0) & (b["prestaged"] == 0)).sum()),
        "large_nd0": int(((rep["nd"] == 0) & (rep["extra"] == 1)).sum()),
    }


# ---------------------------------------------------------------------------------------------------------------------
# host: the replay in the kernel's order
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def host_batch():
    names = list(CLASSES)
    rng = random.Random(90)
    segs = pool(91, 4, [20000, 20480, 65536, 300000, 1 << 20])
    return assemble(rng, segs, runs(rng, names, 2 * len(names)) + pairs(names))


@pytest.mark.parametrize("skew", [0, 5, 15])
def test_replay_in_kernel_order_equals_the_exact_lexer(host_batch, skew):
    docs, cls = host_batch
    tup, toff, _stats, rep = hostsim.warp_batch(docs, skew)
    assert int(toff[-1]) == len(tup)
    for i, doc in enumerate(docs):
        want = hostsim.lex_doc(doc)
        got = tup[int(toff[i]):int(toff[i + 1])]
        if not np.array_equal(got, want):
            raise AssertionError(f"doc {i} ({cls[i]}, skew {skew}, {len(doc)} B) {doc[:120]!r}\n warp ={hostsim.fmt_tuples(got)[:40]}\n"
                                 f" exact={hostsim.fmt_tuples(want)[:40]}")
    h = hand_overs(rep)
    # every hand-over the pipeline has, several times over: the text under each of these writes is the next unit's
    assert h["prestaged_after_deferred"] >= 100, h
    assert h["prestaged_after_fin_cap_write"] >= 20, h
    assert h["prestaged_after_long_line_write"] >= 20, h
    # ... and the units whose writes lex their text again are not staged over
    assert h["staged_after_needs_text"] >= 50, h
    assert h["staged_after_paged"] >= 20, h
    assert h["large_nd0"] >= 15, h
    # nothing skipped the write that needs no text, and every write that needs it kept it
    assert not ((rep["deferred"] == 1) & (rep["needs_text"] == 1)).any()
    assert not ((rep["paged"] == 1) & (rep["needs_text"] == 0)).any()


# ---------------------------------------------------------------------------------------------------------------------
# GPU: at least 8 units per resident warp, every scan organisation, the oracle
# ---------------------------------------------------------------------------------------------------------------------
GPU_LARGE = [20000, 24000, 30000, 40000, 65536, 131072, 400000, 1 << 20]


@pytest.fixture(scope="module")
def gpu_pool():
    segs = pool(92, 6, GPU_LARGE)
    units = {name: [hostsim.warp_units(np.concatenate([[0], np.cumsum([len(d) for d in seg])])) for seg in v] for name, v in segs.items()}
    return segs, units


@pytest.fixture(scope="module")
def scanner():
    import operator_builder_b200 as ob
    sc = ob.Scanner(0)
    yield sc
    sc.set_mode(0)
    sc.close()


def gpu_layout(rng, segs, units, kind, target):
    """segments with at least `target` units in all -> (documents, class of each): runs of 1 to 12, or rounds of every
    class once in random order"""
    names = list(segs)
    picks, have = [], 0
    while have < target:
        for name in (runs(rng, names, len(names)) if kind == "runs" else rng.sample(names, len(names))):
            k = rng.randrange(len(segs[name]))
            picks.append((name, k))
            have += units[name][k]
    if kind == "shuffled":
        rng.shuffle(picks)
    docs, cls = [], []
    for name, k in picks:
        docs += segs[name][k]
        cls += [name] * len(segs[name][k])
    return docs, cls


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["runs", "shuffled"])
def test_many_units_per_warp_on_device(scanner, oracle, gpu_pool, kind):
    import torch
    import operator_builder_b200 as ob
    from operator_builder_b200 import _native
    t0 = time.time()
    segs, units = gpu_pool
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    warps = sms * WPC
    rng = random.Random(93 if kind == "runs" else 94)
    docs, cls = gpu_layout(rng, segs, units, kind, 8 * warps)
    payload = b"".join(docs)
    n, ndocs = len(payload), len(docs)
    off = np.zeros(ndocs + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    nunits = hostsim.warp_units(off)
    assert nunits >= 8 * warps, (nunits, warps)
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    start = 64 + 5  # a base address 5 bytes past a 16-byte boundary
    buf = torch.full((n + 128,), 0x2B, dtype=torch.uint8, device=dev)
    host = np.frombuffer(payload, dtype=np.uint8)
    buf[start:start + n] = torch.from_numpy(host.copy()).to(dev)
    d_bytes = buf.data_ptr() + start
    d_off = torch.from_numpy(off.view(np.int64)).to(dev)

    def scan(mode, cap):
        scanner.set_mode(mode)
        d_out = torch.full((cap + 256,), -1, dtype=torch.int64, device=dev) if cap else None
        d_toff = torch.zeros(ndocs + 1, dtype=torch.int64, device=dev)
        d_status = torch.zeros(4, dtype=torch.int32, device=dev)
        d_counts = torch.zeros(2, dtype=torch.int64, device=dev)
        scanner.lex_batch_device(d_bytes, d_off.data_ptr(), ndocs, n, d_out.data_ptr() if cap else 0, cap, d_toff.data_ptr(),
                                 d_status.data_ptr(), d_counts.data_ptr(), st)
        torch.cuda.synchronize()
        return d_out, d_toff, d_status, d_counts

    _, c_toff, _, _ = scan(1, 0)  # count only (its status[0] says the empty output held nothing): sizes the output exactly
    total = int(c_toff[-1].item())
    ref = scan(0, total)
    out0, toff0, status0, counts0 = ref
    assert int(status0[0].item()) == 0 and int(toff0[-1].item()) == total
    assert (out0[total:] == -1).all()  # nothing written past the tuples
    assert torch.equal(toff0, c_toff)
    for mode in (1, 2, 3, 0):
        out, toff, status, counts = scan(mode, total)
        assert torch.equal(toff, toff0), mode
        assert torch.equal(out, out0), (mode, torch.nonzero(out != out0)[:5].flatten().tolist())
        assert torch.equal(counts, counts0), mode
        # status: overflow, fatal documents, work-record overflow; [1] counts the documents each organisation's exact
        # lexer took, which differs between them by design -- and must not between two runs of one
        keep = [0, 1, 2, 3] if mode == 0 else [0, 2, 3]
        assert torch.equal(status[keep], status0[keep]), (mode, status.tolist(), status0.tolist())
        del out
    scanner.set_mode(0)

    # the oracle: the device hash of every document it models, the decoded stream of the others
    d_hash = torch.zeros(ndocs, dtype=torch.int64, device=dev)
    d_nhost = torch.zeros(1, dtype=torch.int32, device=dev)
    assert _native.lib().obm_hash_batch_device(scanner.handle, d_bytes, d_off.data_ptr(), ndocs, out0.data_ptr(), toff0.data_ptr(),
                                               d_hash.data_ptr(), d_nhost.data_ptr(), st) == 0
    torch.cuda.synchronize()
    got = d_hash.cpu().numpy().view(np.uint64)
    tuples = out0[:total].cpu().numpy().view(np.uint64)
    toff = toff0.cpu().numpy().view(np.uint64)
    del out0, buf
    torch.cuda.empty_cache()
    threads = max(1, len(os.sched_getaffinity(0)))
    _nl, _nm, _h, want = oracle.scan_batch(host, off, threads, want_doc_hash=True)
    left = np.nonzero(got == 0)[0]
    assert len(left) == int(d_nhost.item())
    assert len(left) < ndocs // 4, (len(left), ndocs)
    dev_docs = got != 0
    bad = np.nonzero(dev_docs & (got != want))[0]
    assert len(bad) == 0, [(int(i), cls[i]) for i in bad[:10]]
    sub = [docs[i] for i in left]
    s_off = np.zeros(len(sub) + 1, dtype=np.uint64)
    s_off[1:] = np.cumsum([len(d) for d in sub])
    s_bytes = np.frombuffer(b"".join(sub) + b"\0", dtype=np.uint8)[:-1]
    stream, soff, _nlex = oracle.lex_batch_raw(s_bytes, s_off)
    for k, i in enumerate(left):
        got_i = ob.decode_doc_raw(docs[i], tuples[int(toff[i]):int(toff[i + 1])])
        assert got_i == stream[int(soff[k]):int(soff[k + 1])], (int(i), cls[i], docs[i][:100])
    per_class = {name: sum(1 for x in cls if x == name) for name in CLASSES}
    print(f"\n{kind}: {nunits} units, {ndocs} documents, {n / 1e6:.1f} MB; {warps} resident warps ({sms} SMs x {WPC}): "
          f"{nunits / warps:.1f} units per warp; documents per class {per_class}; {len(left)} documents decoded on the host; "
          f"{time.time() - t0:.1f} s")
