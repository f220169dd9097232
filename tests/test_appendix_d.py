"""SURVEY.md Appendix D: an independent model's outputs (Type, Value, Pos) for 21 inputs that exercise what the
reference's own vectors do not pin -- positions, the stale-buffer prefix (A.4b), column drift (A.6), error and warning
texts, multi-marker lines, a bool literal across a newline.  tools/extract_appendix_d.py transcribes them into
tests/golden/appendix_d.json; here the oracle must reproduce them (CPU) and so must the CUDA path through the C ABI
(GPU).  `<strconv err>` in the survey stands for Go's strconv error text: matched as a wildcard."""
import json
import os
import re

import numpy as np
import pytest

GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "appendix_d.json")))


def same(got, want):
    """got: (type, value bytes, line, col) ; want: [type, value, line, col] with an optional `<strconv err>` wildcard"""
    if got[0] != want[0] or got[2] != want[2] or got[3] != want[3]:
        return False
    val = got[1].decode("utf-8")
    if "<strconv err>" in want[1]:
        pat = "^" + ".*".join(re.escape(p) for p in want[1].split("<strconv err>")) + "$"
        return re.match(pat, val, re.S) is not None and "strconv." in val
    return val == want[1]


def case_id(case):
    """the input's repr, cut to 40 characters; a '::' in it would read as a node-id separator, so its second colon is
    percent-encoded"""
    return repr(case["input"])[:40].replace("::", ":%3A")


@pytest.mark.parametrize("case", GOLD["cases"], ids=[case_id(c) for c in GOLD["cases"]])
def test_oracle_reproduces_appendix_d(oracle, case):
    got = oracle.lex(case["input"].encode())
    assert len(got) == len(case["expected"]), (got, case["expected"])
    for g, w in zip(got, case["expected"]):
        assert same(g, w), (g, w)


def test_host_build_of_the_core_reproduces_appendix_d(oracle):
    from tests import hostsim
    for case in GOLD["cases"]:
        doc = case["input"].encode()
        got = oracle.parse_stream(hostsim.decode(doc, hostsim.lex_doc(doc)))
        assert len(got) == len(case["expected"])
        for g, w in zip(got, case["expected"]):
            assert same(g, w), (doc, g, w)


@pytest.mark.gpu
def test_gpu_reproduces_appendix_d(oracle):
    """every device organisation, through obm_lex_batch, as one packed batch"""
    import operator_builder_b200 as ob
    docs = [c["input"].encode() for c in GOLD["cases"]]
    data = np.frombuffer(b"".join(docs), dtype=np.uint8)
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    sc = ob.Scanner(0)
    try:
        for mode in (0, 1, 2, 3):
            sc.set_mode(mode)
            res = sc.lex_batch(data, off)
            for i, (doc, case) in enumerate(zip(docs, GOLD["cases"])):
                t = res.tuples[int(res.doc_tuple_off[i]):int(res.doc_tuple_off[i + 1])]
                got = oracle.parse_stream(ob.decode_doc_raw(doc, t))
                assert len(got) == len(case["expected"]), (mode, doc)
                for g, w in zip(got, case["expected"]):
                    assert same(g, w), (mode, doc, g, w)
    finally:
        sc.close()
