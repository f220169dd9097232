"""k_warp_scan runs eleven warps per SM (obm_warp.cuh: WPC).  What makes that possible: the unit's packed tuples of the
deferred write (W.fin, FIN_CAP words) live in a per-warp slot in global memory instead of shared memory, and the
registers of eleven warps still fit the SM.

On the host: the shipped library's ptxas report must show k_warp_scan without spills and within the register budget of
WPC warps, and the fixture of the GPU test below must give units whose deferred write fills nearly all of FIN_CAP.
On the GPU: the slots come from each call's scratch, so two scanners that run different batches at the same time on two
streams must not see each other's tuples."""
import os
import random
import re

import numpy as np
import pytest

from tests import hostsim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "operator-builder_b200")
TILE = 12288      # obm_warp.h: a unit = the documents that start in one TILE-byte range of the batch
FIN_CAP = 704     # tuples of a unit whose write is deferred
REGS_PER_SM = 65536


def warps_per_cta():
    src = open(os.path.join(PKG, "csrc", "obm_warp.cuh")).read()
    return int(re.search(r"^#define OBMW_WPC (\d+)$", src, re.M).group(1))


def kernel_report(log, kernel):
    """(registers, spill store bytes, spill load bytes) of `kernel` in a ptxas -v log"""
    m = re.search(r"Function properties for " + re.escape(kernel) + r"\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                  r"(\d+) bytes spill loads\n.*?Used (\d+) registers", log, re.S)
    assert m, f"{kernel} is not in the ptxas report"
    return int(m.group(4)), int(m.group(2)), int(m.group(3))


def test_warp_scan_registers_fit_the_sm_without_spills():
    # the Makefile keeps each library's ptxas report beside it; csrc/build.log is whichever library was built last
    path = os.path.join(PKG, "libobmarkers.so.log")
    assert os.path.exists(path), "build the library first (__graft_entry__.build)"
    regs, st, ld = kernel_report(open(path).read(), "_ZN4obmw11k_warp_scanENS_5WArgsE")
    wpc = warps_per_cta()
    assert wpc >= 11
    assert (regs + 7) // 8 * 8 * 32 * wpc <= REGS_PER_SM, (regs, wpc)
    assert st == 0 and ld == 0, (regs, st, ld)


# ---- a unit whose deferred write fills nearly all of FIN_CAP ---------------------------------------------------------
def plain(rng, n):
    """exactly n bytes (n > 0) of lines without a '#', '+' or "//": no owning line, no tuple but EOF"""
    out = bytearray()
    while len(out) < n - 1:
        out += b"  key%d: value %d\n" % (rng.randrange(1000), rng.randrange(10 ** rng.randint(1, 9)))
    return bytes(out[:n - 1]) + b"\n"


def dense_unit(rng):
    """two 6 KiB documents: 32 staged marker lines of 21 tuples, 13 comment lines of 2 and two EOFs = 700 tuples, all of
    them staged, so the unit takes the deferred write with its slot nearly full"""
    docs = []
    for n_comments in (7, 6):
        lines = [b"# +a:b=%d,c=%d,d=%d,e=%d\n" % tuple(rng.randrange(100) for _ in range(4)) for _ in range(16)]
        lines += [b"# note %d\n" % rng.randrange(10) for _ in range(n_comments)]
        rng.shuffle(lines)
        body = b"k: v\n" + b"".join(lines)
        docs.append(body + plain(rng, TILE // 2 - len(body)))
    return docs


def dense_batch(seed, units):
    rng = random.Random(seed)
    return [d for _ in range(units) for d in dense_unit(rng)]


def offsets(docs):
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    return off


def test_dense_units_take_the_deferred_write_near_fin_cap():
    docs = dense_batch(5, 40)
    tuples, toff, _stats, report = hostsim.warp_batch(docs, skew=3)
    assert len(report) == 40
    assert (report["deferred"][1:] == 1).all() and not report["over_fin"].any() and not report["needs_text"].any()
    per_unit = np.diff(toff.astype(np.int64)[::2])
    assert (per_unit == 700).all(), per_unit
    for i, d in enumerate(docs):
        assert np.array_equal(tuples[int(toff[i]):int(toff[i + 1])], hostsim.lex_doc(d)), i


# ---- GPU: two calls at once, each with its own fin slots -------------------------------------------------------------
@pytest.mark.gpu
def test_concurrent_scans_keep_their_fin_slots_apart():
    import torch
    import operator_builder_b200 as ob
    dev = torch.device("cuda:0")
    warps = torch.cuda.get_device_properties(0).multi_processor_count * warps_per_cta()
    units = 4 * warps  # several units per resident warp: every warp writes its slot many times
    dense = dense_batch(11, units)
    d0, o0 = ob.generate_corpus_host(3 * units, 4096)  # the bench's 4 KiB manifests, three to a unit
    batches = [(np.frombuffer(b"".join(dense), dtype=np.uint8), offsets(dense)), (np.asarray(d0), np.asarray(o0, dtype=np.uint64))]
    assert hostsim.warp_units(batches[0][1]) == units and hostsim.warp_units(batches[1][1]) == units
    dbytes = [torch.from_numpy(b.copy()).to(dev) for b, _ in batches]
    doffs = [torch.from_numpy(o.view(np.int64).copy()).to(dev) for _, o in batches]
    scanners = [ob.Scanner(0), ob.Scanner(0)]
    streams = [torch.cuda.Stream(dev), torch.cuda.Stream(dev)]

    def launch(k, mode, cap, stream):
        sc = scanners[k]
        sc.set_mode(mode)
        ndocs = len(batches[k][1]) - 1
        out = torch.full((cap + 256,), -1, dtype=torch.int64, device=dev)
        toff = torch.zeros(ndocs + 1, dtype=torch.int64, device=dev)
        status = torch.zeros(4, dtype=torch.int32, device=dev)
        counts = torch.zeros(2, dtype=torch.int64, device=dev)
        sc.lex_batch_device(dbytes[k].data_ptr(), doffs[k].data_ptr(), ndocs, int(batches[k][0].size), out.data_ptr(), cap,
                            toff.data_ptr(), status.data_ptr(), counts.data_ptr(), stream.cuda_stream)
        return out, toff, status, counts

    def alone(k, mode, cap):
        r = launch(k, mode, cap, streams[k])
        torch.cuda.synchronize()
        return r

    try:
        torch.cuda.synchronize()
        caps = [int(alone(k, 1, 0)[1][-1].item()) for k in range(2)]
        assert caps[0] == 700 * units
        exact = [alone(k, 1, caps[k]) for k in range(2)]
        single = [alone(k, 0, caps[k]) for k in range(2)]  # also sizes each scanner's scratch, so the calls below allocate nothing
        for k in range(2):
            out, toff, status, counts = single[k]
            assert int(status[0].item()) == 0 and int(toff[-1].item()) == caps[k]
            assert torch.equal(out, exact[k][0]) and torch.equal(toff, exact[k][1]) and torch.equal(counts, exact[k][3]), k
            assert torch.equal(status[[0, 2, 3]], exact[k][2][[0, 2, 3]]), k
        for _ in range(2):
            both = [launch(k, 0, caps[k], streams[k]) for k in range(2)]  # both enqueued before either is waited for
            torch.cuda.synchronize()
            for k in range(2):
                for got, want in zip(both[k], single[k]):
                    assert torch.equal(got, want), k
    finally:
        for sc in scanners:
            sc.close()
