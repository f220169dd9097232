"""The fused warp kernel's unit descriptors (obm_warp.h WUnit, written by k_wunit_descs): one 16-byte load tells a warp
which documents a unit holds and where its text lies.  On the host the table must say what the tile records say
(wrec_unit and the unit's document offsets); on the GPU the scan that reads it must produce the exact path's stream."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

TILE, BUFB, DMAX = 12288, 13312, 31


def doc_of(n, seed):
    """n bytes of manifest-like text with marker lines, newline-terminated (n > 0)"""
    unit = b"# +operator-builder:field:name=f%d,type=string\nkey%d: v # plain\n" % (seed, seed)
    body = (unit * (n // len(unit) + 1))[:n - 1]
    return body + b"\n"


def dense_doc(n, seed):
    """marker-dense: a unit of these has more tuples than the deferred write holds, so it resolves right after publishing"""
    line = b"# +a:b=%d +c:d:e=x,f +g:h='q'\n" % (seed % 10)
    return (line * (n // len(line) + 1))[:n]


def batches():
    small = [doc_of(100, i) for i in range(5)]
    return {
        "split": [doc_of(1500, i) for i in range(9)] + [doc_of(700, 9)] * 4,   # 9 documents start in tile 0, 13,500 bytes: WR_SPLIT
        "large": small + [doc_of(20000, 5)] + small + [doc_of(40000, 6)],    # WR_LARGE; the large documents leave tiles empty
        "only_large": [doc_of(30000, 1)],                                      # a tile whose only unit is the large document
        "dmax": [doc_of(397, i) for i in range(31)] + [doc_of(397, 31)] * 40,  # exactly 31 documents in tile 0, then 31 + 9
        "many_tiny": [doc_of(50, i) for i in range(200)] + [b""] * 40,         # 240 documents per tile: 8 units of it
        "one": [doc_of(3000, 0)],
        "none": [],
    }


def place(payload, skew):
    """payload at a 16k + skew address inside a padded buffer (the device contract: readable around the batch)"""
    buf = np.full(len(payload) + 96, 0x2B, dtype=np.uint8)
    start = (-buf.ctypes.data) % 16 + 16 + (skew & 15)
    buf[start:start + len(payload)] = np.frombuffer(payload, dtype=np.uint8)
    return buf, buf[start:]


def offsets(docs):
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    if docs:
        off[1:] = np.cumsum([len(d) for d in docs])
    return off


@pytest.fixture(scope="module")
def unit_desc_lib(tmp_path_factory):
    """tests/unit_desc_host.cpp: the descriptor code of csrc/obm_warp.h and obm_warp_core.h built for the host"""
    so = str(tmp_path_factory.mktemp("unit_desc") / "libunitdesc.so")
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "unit_desc_host.cpp")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-Wall", "-Wno-unknown-pragmas", "-shared", "-o", so, src])
    return ctypes.CDLL(so)


@pytest.mark.parametrize("name", sorted(batches()))
@pytest.mark.parametrize("skew", [0, 1, 7, 15])
def test_descriptor_table_matches_the_tile_records(unit_desc_lib, name, skew):
    docs = batches()[name]
    off = offsets(docs)
    buf, data = place(b"".join(docs), skew)
    fn = unit_desc_lib.ud_descs
    fn.restype = ctypes.c_uint64
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_uint64]
    cap = 4 * (int(off[-1]) // TILE + 1) + len(docs) + 4
    got = np.zeros((cap, 7), dtype=np.uint64)
    want = np.zeros((cap, 7), dtype=np.uint64)
    n = int(fn(data.ctypes.data, off.ctypes.data, len(docs), got.ctypes.data, want.ctypes.data, cap))
    assert n <= cap and (n > 0) == (len(docs) > 0)
    got, want = got[:n], want[:n]
    assert np.array_equal(got, want), f"first difference at unit {np.argwhere((got != want).any(axis=1))[0][0]}"
    # the units hold every document once, in order: [da, db) and then the large one (extra) at db
    seen = []
    for u, da, db, extra, skw, span, base in got.tolist():
        seen += list(range(da, db)) + ([db] if extra else [])
        if db > da:
            assert span <= BUFB and base % 16 == 0 and base + skw == data.ctypes.data + int(off[da]), (u, da, db)
            assert db - da <= DMAX
    assert seen == list(range(len(docs)))
    nd = got[:, 2] - got[:, 1]
    if name == "dmax":
        assert nd[0] == 31
    if name in ("large", "only_large"):
        assert got[:, 3].sum() >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(batches()) + ["dense"])
@pytest.mark.parametrize("skew", [0, 3, 13])
def test_mode0_stream_equals_the_exact_path(name, skew):
    """k_warp_scan reads the descriptors, prestages the next unit's document offsets and resolves the chain in one round:
    tuple for tuple what the exact path (mode 1) writes, also at bases that are not 16-byte aligned"""
    import torch
    import operator_builder_b200 as ob
    docs = [dense_doc(4096, i) for i in range(300)] + [doc_of(4096, 1)] * 20 + [dense_doc(4096, 7)] * 100 if name == "dense" else batches()[name]
    off = offsets(docs)
    payload = b"".join(docs)
    n, ndocs = len(payload), len(docs)
    dev = torch.device("cuda:0")
    buf = torch.full((n + 128,), 0x2B, dtype=torch.uint8, device=dev)
    start = 64 + skew
    if n:
        buf[start:start + n] = torch.frombuffer(bytearray(payload), dtype=torch.uint8).to(dev)
    d_off = torch.from_numpy(off.astype(np.int64)).to(dev)
    cap = 2 * n + 2 * ndocs + 16
    sc = ob.Scanner(0)
    try:
        res = []
        for mode in (0, 1):
            sc.set_mode(mode)
            d_out = torch.zeros(cap, dtype=torch.int64, device=dev)
            d_toff = torch.zeros(ndocs + 1, dtype=torch.int64, device=dev)
            d_status = torch.zeros(4, dtype=torch.int32, device=dev)
            d_counts = torch.zeros(2, dtype=torch.int64, device=dev)
            sc.lex_batch_device(buf.data_ptr() + start, d_off.data_ptr(), ndocs, n, d_out.data_ptr(), cap, d_toff.data_ptr(),
                                d_status.data_ptr(), d_counts.data_ptr(), torch.cuda.current_stream().cuda_stream)
            torch.cuda.synchronize()
            toff = d_toff.cpu().numpy()
            res.append((d_out[:int(toff[-1])].cpu().numpy(), toff, d_status.cpu().numpy(), d_counts.cpu().numpy()))
        sc.set_mode(0)
    finally:
        sc.close()
    (t0, o0, s0, c0), (t1, o1, s1, c1) = res
    assert s0[0] == 0 and s1[0] == 0  # the output held every tuple
    assert np.array_equal(o0, o1)
    assert np.array_equal(t0, t1), f"first difference at tuple {np.argwhere(t0 != t1)[0][0]}"
    assert np.array_equal(c0, c1)
    if name == "dense":
        assert int(o0[-1]) / (n / TILE) > 704  # a unit has more tuples than the deferred write holds (FIN_CAP)
