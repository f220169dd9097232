"""obm_parse_batch / Scanner.parse_batch: the parser over a HOST batch in one device call -- only the Result records, their
offsets and the tuples of the documents the host parses itself (OBM_R_HOST) come back.

For every document, ParseBatchResult.format_doc must give what parse_doc_raw gives over obm_lex_batch's tuples and what the
parser oracles give (oracle/parser_oracle.py; tests/typed_parser_oracle.py for typed registries); the records must be
bitwise those of obm_parse_batch_device over the same batch (doc_base = 0), whatever the chunking.  Without a GPU, a host
stand-in scanner assembles the same output from tests/hostsim tuples and the host run of the device walk, which covers the
Python side (ParseBatchResult.format_doc, inspect_manifests_parsed)."""
import ctypes
import random

import numpy as np
import pytest

from tests import corpus_util as cu
from tests import hostsim
from tests.test_inspect_batch import compare, manifests, reference_flow
from tests.test_marker_typing import spec, typing_fuzz_doc

F = b"+operator-builder:field"
# one document per outcome the records must carry at least once
OUTCOMES = [b"# +operator-builder:field:name=x,default= true\n",                   # ParseBool error
            b"# +operator-builder:field:name=x,default=1e39\n",                    # float32 range error
            b"# +operator-builder:field:name=x,type=float\n",                      # FieldType unmarshal (typed: SetArgument error)
            b"# +operator-builder:field:name=x\n",                                 # typed: InflateObject, required type missing
            b"# +operator-builder:field:name=1,type=int\n",                        # typed: int for a string field (panic)
            b"# +operator-builder:field:name=a,name=b,type=int\n",                 # typed: last writer wins
            b"# +operator-builder:resource:field=a,value=1,include,include=false\n",
            b"+operator-builder:field:name='unterminated\n"]                        # lexer error: the host parses it
# __graft_entry__.smoke()'s documents: stale buffer, multi-line back-tick, 1e309, text beyond ASCII, pages of owning lines
SMOKE = [b"x: 1+1\n# +a:b=`multi\n  # line`,c\n", b"+a:b=1e309\n# never reached +c:d\n", b"",
         "# café\nk: v # +a:b=1\n".encode(), "# +a:b=é\n".encode(), b"# c\n" * 100,
         b"# +operator-builder:field:name=app.label,type=string,default=\"webstore\"\napp: webstore\n"]
REGISTRIES = ("untyped", "field+collection", "resource")


def registry(kind):
    import operator_builder_b200 as ob
    if kind == "untyped":
        return ob.Registry()
    if kind == "field+collection":
        return ob.Registry.define(ob.FIELD_MARKER, ob.COLLECTION_MARKER)
    return ob.Registry.define(ob.RESOURCE_MARKER)


def corpus(seed=5, n=300):
    import operator_builder_b200 as ob
    rng = random.Random(seed)
    docs = [d for _p, d in cu.fixtures()] + OUTCOMES + SMOKE + list(cu.TARGETED)
    docs += [cu.fuzz_doc(rng) for _ in range(n)] + [cu.fuzz_doc_valid(rng) for _ in range(n)] + [typing_fuzz_doc(rng) for _ in range(2 * n)]
    data0, _ = ob.generate_corpus_host(32, 4096, flavour=0)
    docs += [data0.tobytes()[i * 4096:(i + 1) * 4096] for i in range(32)]
    return docs


def pack(docs, lead=0):
    """docs back to back after `lead` bytes that belong to no document (doc_off[0] = lead)"""
    data = np.frombuffer(b"#" * lead + b"".join(docs) + b"\0", dtype=np.uint8)[:-1]
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    off[0] = lead
    off[1:] = lead + np.cumsum([len(d) for d in docs])
    return data, off


def oracle_results(oracle, kind, doc):
    if kind == "untyped":
        from oracle import parser_oracle as po
    else:
        from tests import typed_parser_oracle as po
    return po.serialize(po.parse(oracle.lex(doc), spec(kind)))


def records_bytes(res):
    return res.results.tobytes(), res.args.tobytes(), res.doc_res_off.tobytes(), res.host_tuples.tobytes(), res.doc_host_off.tobytes()


class HostParseScanner:
    """parse_batch's output assembled on the host: tuples from the host build of the lexer core (tests/hostsim), records
    from the host run of the device walk (obm_parse_doc_records), laid out as obm_parse_batch lays them out"""

    def parse_batch(self, reg, data, off):
        import operator_builder_b200 as ob
        L = ob._native.lib()
        L.obm_parse_doc_records.restype = ctypes.c_int64
        L.obm_parse_doc_records.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p,
                                            ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64)]
        raw = bytes(data)
        rs, ags, hts, roff, hoff = [], [], [], [0], [0]
        nargs_total = 0
        for d in range(len(off) - 1):
            doc = raw[int(off[d]):int(off[d + 1])]
            t = np.ascontiguousarray(hostsim.lex_doc(doc), dtype=np.uint64)
            r = np.zeros(len(t) + 2, dtype=ob.RESULT_DT)
            a = np.zeros(len(t) + 2, dtype=ob.ARG_DT)
            na = ctypes.c_uint64()
            n = L.obm_parse_doc_records(reg.handle, doc, t.ctypes.data, len(t), d, r.ctypes.data, len(r), a.ctypes.data, len(a), ctypes.byref(na))
            assert n >= 0
            r = r[:n]
            host = n == 1 and (int(r[0]["flags"]) & ob.lexer.R_HOST) != 0
            r["arg_base"] = np.where(r["flags"] & ob.lexer.R_HOST, r["arg_base"], r["arg_base"] + nargs_total)
            rs.append(r); ags.append(a[:na.value]); hts.append(t if host else t[:0])
            nargs_total += int(na.value)
            roff.append(roff[-1] + n); hoff.append(hoff[-1] + (len(t) if host else 0))
        cat = lambda xs, dt: np.concatenate(xs) if xs else np.zeros(0, dt)  # noqa: E731
        return ob.ParseBatchResult(reg, cat(rs, ob.RESULT_DT), cat(ags, ob.ARG_DT), np.array(roff, np.uint64), cat(hts, np.uint64),
                                   np.array(hoff, np.uint64), {})


def test_host_assembly_format_doc_and_inspection(oracle):
    """the Python assembly without a GPU: format_doc over parse_batch's layout == the parser oracles; the inspection from one
    parse_batch == the reference's per-node flow"""
    import operator_builder_b200 as ob
    from operator_builder_b200 import inspect as ins
    docs = corpus(n=60)
    data, off = pack(docs, lead=3)
    sc = HostParseScanner()
    n_host = 0
    for kind in REGISTRIES:
        res = sc.parse_batch(registry(kind), data, off)
        for d, doc in enumerate(docs):
            assert res.format_doc(d, doc) == oracle_results(oracle, kind, doc), (kind, d, doc)
        n_host += int(res.doc_host_off[-1] > 0)
    assert n_host == len(REGISTRIES)
    mans = manifests()
    assert compare(ins.inspect_manifests_parsed(sc, ob.Registry(), mans), reference_flow(oracle, mans)) >= 60


# ---- on the GPU ------------------------------------------------------------------------------------------------------
def device_records(sc, reg, data, off, lexed):
    """obm_lex_batch_device + obm_parse_batch_device (doc_base 0) over a device copy of the batch -> host arrays"""
    import torch
    dev = torch.device("cuda:0")
    base = int(off[0])
    d_bytes = torch.zeros(max(len(data) - base, 1) + 16, dtype=torch.uint8, device=dev)
    if len(data) > base:
        d_bytes[:len(data) - base] = torch.from_numpy(np.array(data[base:], dtype=np.uint8)).to(dev)
    d_off = torch.from_numpy((off - off[0]).astype(np.int64)).to(dev)
    ndocs = len(off) - 1
    cap = max(len(lexed.tuples), 1)
    d_tup = torch.zeros(cap, dtype=torch.int64, device=dev)
    d_toff = torch.zeros(ndocs + 1, dtype=torch.int64, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    sc.lex_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, int(off[-1] - off[0]), d_tup.data_ptr(), cap, d_toff.data_ptr(), stream=st)
    d_res = torch.zeros(cap * 32, dtype=torch.uint8, device=dev)
    d_args = torch.zeros(cap * 16, dtype=torch.uint8, device=dev)
    d_roff = torch.zeros(ndocs + 1, dtype=torch.int64, device=dev)
    d_tot = torch.zeros(2, dtype=torch.int64, device=dev)
    sc.parse_batch_device(reg, d_bytes.data_ptr(), d_off.data_ptr(), ndocs, 0, d_tup.data_ptr(), d_toff.data_ptr(), d_res.data_ptr(), cap,
                          d_args.data_ptr(), cap, d_roff.data_ptr(), d_tot.data_ptr(), stream=st)
    torch.cuda.synchronize()
    nres, nargs = [int(x) for x in d_tot.cpu().tolist()]
    assert np.array_equal(d_toff.cpu().numpy().view(np.uint64), lexed.doc_tuple_off)
    return d_res.cpu().numpy()[:nres * 32].tobytes(), d_args.cpu().numpy()[:nargs * 16].tobytes(), d_roff.cpu().numpy().view(np.uint64)


def check_against_lex(res, lexed, docs):
    """fallback tuples: exactly obm_lex_batch's tuples of the R_HOST documents, nothing for the others"""
    import operator_builder_b200 as ob
    for d in range(len(docs)):
        r = res.results[int(res.doc_res_off[d]):int(res.doc_res_off[d + 1])]
        t = lexed.tuples[int(lexed.doc_tuple_off[d]):int(lexed.doc_tuple_off[d + 1])]
        h = res.host_tuples[int(res.doc_host_off[d]):int(res.doc_host_off[d + 1])]
        assert (r["doc"] == d).all()
        if len(r) == 1 and int(r[0]["flags"]) & ob.lexer.R_HOST:
            assert np.array_equal(h, t), d
        else:
            assert len(h) == 0, d


@pytest.mark.gpu
def test_parse_batch_equals_oracles_and_device_call(oracle):
    import operator_builder_b200 as ob
    from operator_builder_b200 import lexer as lx
    docs = corpus()
    data, off = pack(docs)
    sc = ob.Scanner(0)
    lexed = sc.lex_batch(data, off)
    seen_flags, seen_arg_flags = 0, 0
    try:
        for kind in REGISTRIES:
            reg = registry(kind)
            res = sc.parse_batch(reg, data, off)
            assert sc._L.obm_launches_last_call(sc.handle) > 0
            for d, doc in enumerate(docs):
                got = res.format_doc(d, doc)
                t = lexed.tuples[int(lexed.doc_tuple_off[d]):int(lexed.doc_tuple_off[d + 1])]
                assert got == ob.parse_doc_raw(reg, doc, t) == oracle_results(oracle, kind, doc), (kind, d, doc)
            check_against_lex(res, lexed, docs)
            R, A, roff = device_records(sc, reg, data, off, lexed)
            assert res.results.tobytes() == R and res.args.tobytes() == A and np.array_equal(res.doc_res_off, roff), kind
            assert res.stats["n_tuples"] == len(lexed.tuples) and res.stats["bytes"] == len(data)
            seen_flags |= int(np.bitwise_or.reduce(res.results["flags"]))
            seen_arg_flags |= int(np.bitwise_or.reduce(res.args["flags"]))
    finally:
        sc.close()
    for f in (lx.R_HOST, lx.R_ERR_PARSEBOOL, lx.R_ERR_FLOAT32, lx.R_ERR_SETARG, lx.R_ERR_MISSING, lx.R_PANIC):
        assert seen_flags & f, f
    assert seen_arg_flags & lx.A_SUPERSEDED


@pytest.mark.gpu
def test_parse_batch_chunked_equals_single_shot(oracle):
    """many 4 KiB chunks through the three-slot pipeline: a document larger than a chunk, one over 13,296 bytes (the large
    document path), empty documents, doc_off[0] != 0 -- the same bytes as one chunk, with global doc ids and arg_base"""
    import operator_builder_b200 as ob
    big = b"".join(b"# +operator-builder:field:name=f%d,type=int,default=%d\nk%d: v\n" % (i, i, i) for i in range(400))
    assert len(big) > 13296
    mid = b"# filler\n" * 600 + b"# +operator-builder:field:name=m,type=string\n"
    docs = corpus(seed=9, n=150)
    docs = docs[:40] + [b"", big, b""] + docs[40:200] + [mid, b""] + docs[200:]
    data, off = pack(docs, lead=5)
    sc = ob.Scanner(0)
    try:
        lexed = sc.lex_batch(data, off)
        for kind in REGISTRIES:
            reg = registry(kind)
            one = sc.parse_batch(reg, data, off)
            sc.set_chunk_bytes(4096)
            many = sc.parse_batch(reg, data, off)
            launches = sc._L.obm_launches_last_call(sc.handle)
            sc.set_chunk_bytes(64 << 20)
            assert records_bytes(many) == records_bytes(one), kind
            assert launches > 40
            check_against_lex(many, lexed, docs)
            R, A, roff = device_records(sc, reg, data, off, lexed)
            assert many.results.tobytes() == R and many.args.tobytes() == A and np.array_equal(many.doc_res_off, roff), kind
            ok = many.results[(many.results["flags"] & ob.lexer.R_HOST) == 0]
            # arg_base indexes the whole batch's args (check_against_lex: every record's doc is its global index)
            ends = ok["arg_base"].astype(np.int64) + ok["nargs"]
            assert (np.diff(ok["arg_base"].astype(np.int64)) >= 0).all() and int(ends.max()) <= len(many.args) and int(ends.max()) > len(many.args) // 2
            for d, doc in enumerate(docs):
                assert many.format_doc(d, doc) == oracle_results(oracle, kind, doc), (kind, d)
            assert many.stats["n_tuples"] == len(lexed.tuples)
    finally:
        sc.close()


def raw_parse(sc, reg, data, off, res=None, res_cap=0, args=None, arg_cap=0, host=None, host_cap=0):
    ndocs = len(off) - 1
    roff = np.full(ndocs + 1, 7, np.uint64); hoff = np.full(ndocs + 1, 7, np.uint64); tot = np.zeros(3, np.uint64)
    p = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
    buf = data if len(data) else np.zeros(1, np.uint8)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    rc = sc._L.obm_parse_batch(sc.handle, reg.handle, buf.ctypes.data, off.ctypes.data, ndocs, p(res), res_cap, p(args), arg_cap,
                               roff.ctypes.data, p(host), host_cap, hoff.ctypes.data, tot.ctypes.data, None)
    return rc, [int(x) for x in tot], roff, hoff


@pytest.mark.gpu
def test_parse_batch_capacities_and_arguments():
    import operator_builder_b200 as ob
    from operator_builder_b200 import _native
    docs = corpus(seed=13, n=100)
    data, off = pack(docs)
    sc = ob.Scanner(0)
    try:
        reg = registry("field+collection")
        for chunk in (64 << 20, 4096):
            sc.set_chunk_bytes(chunk)
            rc, tot, roff, hoff = raw_parse(sc, reg, data, off)  # the NULL sizing call
            assert rc == _native.OBM_E_CAPACITY and min(tot) > 0
            full = sc.parse_batch(reg, data, off)
            assert tot == [len(full.results), len(full.args), len(full.host_tuples)]
            assert np.array_equal(roff, full.doc_res_off) and np.array_equal(hoff, full.doc_host_off)
            for short in range(3):
                caps = [t - (i == short) for i, t in enumerate(tot)]
                SENT = 64
                res = np.zeros(caps[0] + SENT, ob.RESULT_DT); res.view(np.uint8)[:] = 0xAB
                args = np.zeros(caps[1] + SENT, ob.ARG_DT); args.view(np.uint8)[:] = 0xAB
                host = np.full(caps[2] + SENT, 0xABABABABABABABAB, np.uint64)
                rc, got, roff, hoff = raw_parse(sc, reg, data, off, res, caps[0], args, caps[1], host, caps[2])
                assert rc == _native.OBM_E_CAPACITY and got == tot, (chunk, short)
                assert np.array_equal(roff, full.doc_res_off) and np.array_equal(hoff, full.doc_host_off)
                assert (res.view(np.uint8)[caps[0] * 32:] == 0xAB).all()
                assert (args.view(np.uint8)[caps[1] * 16:] == 0xAB).all()
                assert (host[caps[2]:] == 0xABABABABABABABAB).all()
            with pytest.raises(ob.NativeError):
                sc.parse_batch(reg, data, off, res_cap=tot[0], arg_cap=tot[1], host_cap=tot[2] - 1)
        sc.set_chunk_bytes(64 << 20)
        rc, tot, roff, hoff = raw_parse(sc, reg, np.zeros(0, np.uint8), np.zeros(1, np.uint64))
        assert rc == 0 and tot == [0, 0, 0] and roff[0] == 0 and hoff[0] == 0
        empty = sc.parse_batch(reg, np.zeros(0, np.uint8), np.zeros(1, np.uint64))
        assert len(empty.results) == 0 and list(empty.doc_res_off) == [0]
        nine = ob.Registry({b"+m%d:x" % i: [b"a"] for i in range(9)})
        assert raw_parse(sc, nine, data, off)[0] == _native.OBM_E_ARG
        bad = off.copy(); bad[3], bad[4] = bad[4], bad[3]
        assert raw_parse(sc, reg, data, bad)[0] == _native.OBM_E_ARG
    finally:
        sc.close()


@pytest.mark.gpu
def test_parse_batch_1gib_equals_device_call():
    """262,144 generated 4 KiB documents (1 GiB, BASELINE.md C2) through the chunked host call: records bitwise those of
    obm_parse_batch_device over the device-resident copy"""
    import operator_builder_b200 as ob
    data, off = ob.generate_corpus_host(262144, 4096, flavour=0)
    sc = ob.Scanner(0)
    try:
        reg = ob.Registry()
        res = sc.parse_batch(reg, data, off)
        assert len(res.results) > 262144 * 4
        import torch
        dev = torch.device("cuda:0")
        d_bytes = torch.from_numpy(data).to(dev)
        d_off = torch.from_numpy(off.astype(np.int64)).to(dev)
        cap = int(res.stats["n_tuples"])
        d_tup = torch.empty(cap, dtype=torch.int64, device=dev)
        d_toff = torch.empty(len(off), dtype=torch.int64, device=dev)
        st = torch.cuda.current_stream().cuda_stream
        sc.lex_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), 262144, len(data), d_tup.data_ptr(), cap, d_toff.data_ptr(), stream=st)
        d_res = torch.empty(len(res.results) * 32, dtype=torch.uint8, device=dev)
        d_args = torch.empty(len(res.args) * 16, dtype=torch.uint8, device=dev)
        d_roff = torch.empty(len(off), dtype=torch.int64, device=dev)
        d_tot = torch.zeros(2, dtype=torch.int64, device=dev)
        sc.parse_batch_device(reg, d_bytes.data_ptr(), d_off.data_ptr(), 262144, 0, d_tup.data_ptr(), d_toff.data_ptr(), d_res.data_ptr(),
                              len(res.results), d_args.data_ptr(), len(res.args), d_roff.data_ptr(), d_tot.data_ptr(), stream=st)
        torch.cuda.synchronize()
        assert [int(x) for x in d_tot.cpu().tolist()] == [len(res.results), len(res.args)]
        assert d_res.cpu().numpy().tobytes() == res.results.tobytes()
        assert d_args.cpu().numpy().tobytes() == res.args.tobytes()
        assert np.array_equal(d_roff.cpu().numpy().view(np.uint64), res.doc_res_off)
    finally:
        sc.close()


@pytest.mark.gpu
def test_inspection_from_one_parse_batch(oracle):
    import operator_builder_b200 as ob
    from operator_builder_b200 import inspect as ins
    mans = manifests()
    sc = ob.Scanner(0)
    try:
        got = ins.inspect_manifests_parsed(sc, ob.Registry(), mans)
    finally:
        sc.close()
    assert compare(got, reference_flow(oracle, mans)) >= 60
