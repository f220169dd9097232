"""Typed marker arguments: Definition.SetArgument -> Argument.SetValue (internal/markers/marker/argument.go:91-127,
marker.go:53-63) and InflateObject (marker.go:65-95) for the three definitions operator-builder registers
(internal/workload/v1/markers: field_marker.go:26-38, resource_marker.go:47-57).

Three implementations must agree byte for byte: tests/typed_parser_oracle.py (the parser oracle with typed definitions,
OPERATOR_BUILDER_TYPED) over the oracle lexer,
the host mirror obm_parse_doc, and the device walk (csrc/obm_parse_dev.h, parse_doc<true>) run on the host through
obm_parse_doc_records + obm_results_format_doc; on the GPU, k_parse_docs<., true> as well.  The outcome class of every
SetArgument is also checked against a table written here from the Go spec's conversion / assignability rules.  Parity
unpinned (the reference has no parser tests) except the FieldType names (tests/golden/field_types.json)."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

from tests import corpus_util as cu
from tests import hostsim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES_DT = np.dtype([("doc", "<u4"), ("tuple", "<u4"), ("text_off", "<u4"), ("text_len", "<u4"), ("reg_id", "<u2"), ("nargs", "<u2"),
                   ("arg_base", "<u4"), ("flags", "<u4"), ("aux", "<u4")])
ARG_DT = np.dtype([("name_off", "<u4"), ("val_off", "<u4"), ("val_len", "<u4"), ("name_len", "<u2"), ("kind", "u1"), ("flags", "u1")])
R_OK, R_HOST, R_ERR_SETARG, R_ERR_MISSING, R_PANIC = 1, 16, 32, 64, 128
A_SUPERSEDED = 2
F = b"+operator-builder:field"
C = b"+operator-builder:collection:field"
R = b"+operator-builder:resource"

_REGS = {}


def reg(kind="typed"):
    """registries by name, built once: 'typed' = all three typed definitions, 'untyped' = the names-only one"""
    if kind not in _REGS:
        import operator_builder_b200 as ob
        if kind == "typed":
            _REGS[kind] = ob.Registry.define(ob.FIELD_MARKER, ob.COLLECTION_MARKER, ob.RESOURCE_MARKER)
        elif kind == "untyped":
            _REGS[kind] = ob.Registry()
        elif kind == "resource":
            _REGS[kind] = ob.Registry.define(ob.RESOURCE_MARKER)
        elif kind == "field+collection":
            _REGS[kind] = ob.Registry.define(ob.FIELD_MARKER, ob.COLLECTION_MARKER)
        elif kind == "mixed":  # untyped field marker, typed resource marker, an untyped marker of another tool
            _REGS[kind] = ob.Registry({F: [b"name", b"type", b"description", b"default", b"replace"], b"+kubebuilder:validation": [b"Enum"]})
            _REGS[kind].define_marker(ob.RESOURCE_MARKER)
    return _REGS[kind]


def spec(kind="typed"):
    from oracle import parser_oracle
    from tests import typed_parser_oracle as po
    T, U = po.OPERATOR_BUILDER_TYPED, parser_oracle.OPERATOR_BUILDER_REGISTRY
    return {"typed": T, "untyped": U, "resource": {R: T[R]}, "field+collection": {F: T[F], C: T[C]},
            "mixed": {F: U[F], b"+kubebuilder:validation": {b"Enum"}, R: T[R]}}[kind]


def _lib():
    import operator_builder_b200 as ob
    L = ob._native.lib()
    L.obm_parse_doc_records.restype = ctypes.c_int64
    L.obm_parse_doc_records.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_uint32, ctypes.c_void_p,
                                        ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64, ctypes.POINTER(ctypes.c_uint64)]
    L.obm_results_format_doc.restype = ctypes.c_int64
    L.obm_results_format_doc.argtypes = [ctypes.c_void_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_uint64, ctypes.c_void_p,
                                         ctypes.c_uint64, ctypes.c_void_p, ctypes.POINTER(ctypes.POINTER(ctypes.c_uint8)), ctypes.POINTER(ctypes.c_uint64)]
    return L


def walk_records(r, doc, tuples, doc_id=0):
    """the device walk on the host: (results, arguments) as k_parse_docs writes them for this one document"""
    L = _lib()
    tuples = np.ascontiguousarray(tuples, dtype=np.uint64)
    res = np.zeros(len(tuples) + 2, dtype=RES_DT); args = np.zeros(len(tuples) + 2, dtype=ARG_DT)
    na = ctypes.c_uint64()
    n = L.obm_parse_doc_records(r.handle, doc, tuples.ctypes.data, len(tuples), doc_id, res.ctypes.data, len(res), args.ctypes.data, len(args),
                                ctypes.byref(na))
    assert n >= 0
    return res[:n], args[:na.value]


def format_records(r, doc, tuples, res, args):
    L = _lib()
    tuples = np.ascontiguousarray(tuples, dtype=np.uint64)
    res = np.ascontiguousarray(res); args = np.ascontiguousarray(args)
    out = ctypes.POINTER(ctypes.c_uint8)(); outlen = ctypes.c_uint64()
    n = L.obm_results_format_doc(r.handle, doc, len(doc), tuples.ctypes.data, len(tuples), res.ctypes.data, len(res),
                                 args.ctypes.data if len(args) else None, ctypes.byref(out), ctypes.byref(outlen))
    assert n >= 0
    data = ctypes.string_at(out, outlen.value)
    L.obm_free(out)
    return data


def check(oracle, doc, kind="typed", tuples=None):
    """oracle == obm_parse_doc == the device walk (host run); returns the oracle's Results"""
    import operator_builder_b200 as ob
    from tests import typed_parser_oracle as po
    results = po.parse(oracle.lex(doc), spec(kind))
    want = po.serialize(results)
    tuples = hostsim.lex_doc(doc) if tuples is None else tuples
    got = ob.parse_doc_raw(reg(kind), doc, tuples)
    assert got == want, (doc, got, want)
    res, args = walk_records(reg(kind), doc, tuples)
    dev = format_records(reg(kind), doc, tuples, res, args)
    assert dev == want, (doc, dev, want)
    return results


# ---- the SetArgument matrix --------------------------------------------------------------------------------------------
# value forms -> the Go value type parseArgValue passes (state.go:95-153); the lexer makes bool literals of "true" and "false"
# only (lexer/state.go:279), so "False" is a naked string
FORMS = [(b"", "bool"), (b"=true", "bool"), (b"=False", "string"), (b"=1", "int"), (b"=-0", "int"), (b"=007", "int"), (b"=1.5", "float64"),
         (b"=0.1", "float64"), (b"=1e6", "float64"), (b'="s"', "string"), (b"=s", "string"), (b"=''", "string"), (b"=`b`", "string")]
# the Go type of every argument (field_marker.go:26-38, resource_marker.go:47-57)
ARG_TYPES = {F: {b"name": "string", b"type": "FieldType", b"description": "*string", b"default": "interface{}", b"replace": "*string"},
             R: {b"field": "*string", b"collectionField": "*string", b"value": "interface{}", b"include": "*bool"}}
ARG_TYPES[C] = ARG_TYPES[F]
PREFIX = {F: b"name=n,type=int,", C: b"name=n,type=int,", R: b"value=1,"}  # the required arguments, set before the one under test


def expected_class(gotype, vtype):
    """Go spec: a value converts to an identical type, to interface{} and, from an integer, to a string type; reflect.Value.Set
    needs assignability (identical, or interface{}).  FieldType takes the UnmarshalMarkerArg branch and needs a string."""
    if gotype == "FieldType":
        return "unmarshal" if vtype == "string" else "not-a-string"  # none of the string forms is a FieldType name
    elem = gotype.lstrip("*")
    if elem == "interface{}" or vtype == elem:
        return "ok"
    if vtype == "int" and elem == "string":
        return "panic"
    return "wrong-type"


def outcome_class(results):
    last = results[-1]
    if last[0] == "ok":
        return "ok"
    if last[0] == "panic":
        return "panic"
    msg = last[1]
    if msg.startswith("incorrect type, wanted "):
        return "wrong-type"
    if msg.startswith("unable to unmarshal arg value, cannot convert "):
        return "not-a-string"
    if msg.startswith('unable to unmarshal arg value "'):
        return "unmarshal"
    return msg


def test_setargument_matrix(oracle):
    n = 0
    for marker, args in ARG_TYPES.items():
        for arg, gotype in args.items():
            for form, vtype in FORMS:
                doc = b"# " + marker + b":" + PREFIX[marker] + arg + form + b"\n"
                results = check(oracle, doc)
                assert len(results) == 1, (doc, results)
                assert outcome_class(results) == expected_class(gotype, vtype), (doc, results)
                n += 1
    assert n == 14 * len(FORMS)


def test_message_texts(oracle):
    """the exact texts, including %v of each Go value"""
    cases = {
        b"+operator-builder:field:name=replicas,type=strin":
            'unable to unmarshal arg value "strin", unable to parse field, strin into FieldType on arg type, on marker +operator-builder:field at {line:1 column:44}',
        b"+operator-builder:field:name=a,type=007": "unable to unmarshal arg value, cannot convert 7 to string on arg type, on marker +operator-builder:field at {line:1 column:37}",
        b"+operator-builder:field:name=a,type=-0": "unable to unmarshal arg value, cannot convert 0 to string on arg type",
        b"+operator-builder:field:name=a,type=true": "unable to unmarshal arg value, cannot convert true to string on arg type",
        b"+operator-builder:field:name=a,type=0.1": "unable to unmarshal arg value, cannot convert 0.10000000149011612 to string on arg type",
        b"+operator-builder:field:name=a,type=1e6": "unable to unmarshal arg value, cannot convert 1e+06 to string on arg type",   # unpinned: %g rule
        b"+operator-builder:field:name=a,type=100000.0": "unable to unmarshal arg value, cannot convert 100000 to string on arg type",  # unpinned
        b"+operator-builder:field:name=a,type=''": 'unable to unmarshal arg value "", unable to parse field,  into FieldType on arg type',
        b"+operator-builder:resource:value=1,include=1": 'incorrect type, wanted "bool" but received "int" on arg include',
        b"+operator-builder:resource:value=1,field=true": 'incorrect type, wanted "string" but received "bool" on arg field',
        b"+operator-builder:field:name=1.5,type=int": 'incorrect type, wanted "string" but received "float64" on arg name',
    }
    for doc, msg in cases.items():
        results = check(oracle, doc)
        assert results[-1][0] == "error" and results[-1][1].startswith(msg), (doc, results)
    results = check(oracle, b"+operator-builder:field:name=1,type=int")
    assert results == [("panic", "reflect.Set: value of type int is not assignable to type string", b"+operator-builder:field:name=1")]


def test_float_formatting_powers_of_two(oracle):
    """%v of float32 values widened to float64: the host formatter against the oracle's, at every power of two float32 holds
    (where the shortest decimal's rounding interval is lopsided) and a sweep of ordinary values"""
    from tests import typed_parser_oracle as po
    vals = [f"{2.0 ** e!r}".encode() for e in range(-149, 128)] + [b"%de%d" % (m, e) for m in (1, 3, 7, 12345, 99999) for e in range(-44, 34, 3)]
    for v in vals:
        doc = b"+operator-builder:field:name=a,type=" + v
        if po.read_float_magnitude(v) >= po.F32_OVERFLOW_DEC or b"." not in v and b"e" not in v:
            continue
        check(oracle, doc)


def load_field_types():
    with open(os.path.join(ROOT, "tests", "golden", "field_types.json")) as f:
        return json.load(f)


def test_field_type_vectors(oracle):
    """field_types_internal_test.go:12-93 (pinned) plus near misses"""
    g = load_field_types()
    assert len(g["cases"]) == 6
    for c in g["cases"] + [{"in": "String", "wantErr": True}, {"in": "int ", "wantErr": True}, {"in": "strin", "wantErr": True},
                           {"in": "bool", "wantErr": False}]:
        doc = b'# +operator-builder:collection:field:name=n,type="' + c["in"].encode() + b'"\n'
        results = check(oracle, doc)
        assert (results[-1][0] == "error") == c["wantErr"], (c, results)
        if not c["wantErr"]:
            assert dict(results[-1][4])[b"type"] == ("string", c["in"].encode())


def test_missing_arguments(oracle):
    for doc, missing in [(b"+operator-builder:field:name=a", ['"type"']), (b"+operator-builder:field:type=int", ['"name"']),
                         (b"+operator-builder:field:description=d", ['"name"', '"type"']),
                         (b"+operator-builder:collection:field:default=1,replace=r", ['"name"', '"type"']),
                         (b"+operator-builder:resource:field=a,include", ['"value"'])]:
        results = check(oracle, doc + b"\n")
        (kind, msg, text), = results
        assert kind == "error" and text == doc + b"\n"
        head, pos = msg.split(", on marker ")
        assert pos.endswith(" at {line:0 column:0}")
        assert head.startswith("unable to inflate object, missing arguments: [") and head.endswith("]")
        assert sorted(head[len("unable to inflate object, missing arguments: ["):-1].split(" ")) == sorted(missing)  # Go: map order
    res, _a = walk_records(reg(), b"+operator-builder:field:description=d\n", hostsim.lex_doc(b"+operator-builder:field:description=d\n"))
    assert len(res) == 1 and int(res[0]["flags"]) == R_ERR_MISSING | 2 and int(res[0]["aux"]) == 3 and int(res[0]["nargs"]) == 0


def test_duplicates_last_writer_wins(oracle):
    doc = b"+operator-builder:field:name=a,type=int,name=b,type=bool,name=c\n"
    results = check(oracle, doc)
    assert results[0][0] == "ok" and dict(results[0][4])[b"name"] == ("string", b"c") and dict(results[0][4])[b"type"] == ("string", b"bool")
    res, args = walk_records(reg(), doc, hostsim.lex_doc(doc))
    assert [int(a["flags"]) & A_SUPERSEDED for a in args] == [2, 2, 2, 0, 0]
    # good then bad: the error; bad then good: the error at the first
    r = check(oracle, b"+operator-builder:field:name=a,type=int,type=strin\n")
    assert r[-1][0] == "error" and "arg type" in r[-1][1]
    r = check(oracle, b"+operator-builder:field:name=a,type=strin,type=int\n")
    assert r[-1][0] == "error" and "strin" in r[-1][1] and r[-1][2] == b"+operator-builder:field:name=a,type=strin"
    # untyped definitions never mark superseded arguments
    res, args = walk_records(reg("untyped"), doc, hostsim.lex_doc(doc))
    assert not any(int(a["flags"]) & A_SUPERSEDED for a in args)


def test_failure_in_second_marker(oracle):
    for bad in (b"type=strin", b"name=1", b"description=d", b"replace=1.5"):
        doc = (b"# +operator-builder:field:name=a,type=int\n# +operator-builder:field:name=b," + bad +
               b"\n# +operator-builder:resource:value=1\n")
        results = check(oracle, doc)
        assert len(results) == 2 and results[0][0] == "ok" and results[1][0] in ("error", "panic"), (doc, results)


def _col(doc, line, needle):
    return doc.split(b"\n")[line - 1].index(needle) + 1


def test_error_positions(oracle):
    # a synthetic true is peeked, not consumed: parser.current is the Arg (or the ArgAssignment after it); MarkerText stops before it
    doc = b"x\n  # +operator-builder:field:name=a,type\n"
    r = check(oracle, doc)
    assert r[-1][1].endswith("at {line:2 column:%d}" % _col(doc, 2, b"type")) and r[-1][2] == b"+operator-builder:field:name=a,type"
    doc = b"+operator-builder:field:name=a,type,description=d\n"  # the synthetic true before a delimiter
    r = check(oracle, doc)
    assert "cannot convert true" in r[-1][1] and r[-1][2] == b"+operator-builder:field:name=a,type"
    assert r[-1][1].endswith("at {line:1 column:%d}" % _col(doc, 1, b"type"))
    doc = b"+operator-builder:resource:value=2,field,include\n"
    r = check(oracle, doc)
    assert r[-1][1].endswith("at {line:1 column:%d}" % _col(doc, 1, b"field,"))
    # literals: parser.current is the literal
    doc = b"\n\n   +operator-builder:resource:value=2,include=1.5\n"
    r = check(oracle, doc)
    assert r[-1][1].endswith("at {line:3 column:%d}" % _col(doc, 3, b"1.5")) and r[-1][2].endswith(b"include=1.5")
    doc = b'+operator-builder:field:name=a,type="flt"\n'
    r = check(oracle, doc)
    assert r[-1][1].endswith("at {line:1 column:%d}" % _col(doc, 1, b"flt")) and r[-1][2].endswith(b'type="flt')


def test_subset_and_mixed_registries(oracle):
    docs = [b"+operator-builder:field:name=1,type=int\n+operator-builder:resource:value=1,include=1\n",
            b"+operator-builder:resource:include\n+operator-builder:field:type=int\n",
            b"+operator-builder:collection:field:type=x\n+operator-builder:field:name=1,type=int\n",
            b"+kubebuilder:validation:Enum=1\n+operator-builder:field:name=1,type=1\n+operator-builder:resource:field=a\n"]
    for kind in ("resource", "field+collection", "mixed", "untyped"):
        for doc in docs:
            check(oracle, doc, kind)
    assert check(oracle, docs[0], "resource")[-1][1].startswith('incorrect type, wanted "bool"')
    assert check(oracle, docs[1], "field+collection")[-1][1].startswith("unable to inflate object")
    assert check(oracle, docs[3], "mixed")[-1][1].startswith("unable to inflate object, missing arguments: [\"value\"]")


TYPING_ARGS = [b"name", b"type", b"description", b"default", b"replace", b"field", b"collectionField", b"value", b"include", b"bogus"]
TYPING_VALUES = [form for form, _v in FORMS] + [b"=int", b"=string", b"=bool", b"=strin", b"=T", b"=1e39", b"= true", b'="a b"', b"=`x\n# y`"]
TYPING_MARKERS = [F, C, R, b"+kubebuilder:validation", b"+operator-builder:fieldx"]


def typing_fuzz_doc(rng):
    """lines of markers with arguments drawn from all three definitions and values of every kind, mostly well formed: biased
    toward the SetArgument / InflateObject outcomes rather than the lexer's"""
    lines = []
    for _ in range(rng.randint(1, 4)):
        marker = rng.choice(TYPING_MARKERS)
        args = [PREFIX[marker]] if marker in PREFIX and rng.random() < 0.6 else []
        args += [rng.choice(TYPING_ARGS) + rng.choice(TYPING_VALUES) + b"," for _ in range(rng.randint(0, 3))]
        body = b"".join(args).rstrip(b",") or b"name=x"
        lines.append(rng.choice([b"# ", b"", b"  # x ", b"- a: 1 # "]) + marker + b":" + body)
    return b"\n".join(lines) + rng.choice([b"\n", b""])


def test_typing_fuzz(oracle):
    rng = random.Random(4091)
    kinds = {"ok": 0, "error": 0, "panic": 0}
    for i in range(3000):
        results = check(oracle, typing_fuzz_doc(rng), ("typed", "resource", "mixed")[i % 3])
        for r in results:
            kinds[r[0]] += 1
    for _ in range(300):
        check(oracle, cu.fuzz_doc_valid(rng))
    assert min(kinds.values()) > 20, kinds


def test_fixtures_and_generated_batch_typed_equals_untyped(oracle):
    """the reference's fixtures, and C2-style generated documents: the generator writes only well-typed markers
    (obm_corpus.h:6-11), so the typed walk writes the untyped walk's records -- no error records, nothing superseded"""
    import operator_builder_b200 as ob
    for _p, doc in cu.fixtures():
        check(oracle, doc)
    data0, _ = ob.generate_corpus_host(200, 4096, flavour=0)
    n_ok = 0
    for i in range(200):
        doc = data0.tobytes()[i * 4096:(i + 1) * 4096]
        t = hostsim.lex_doc(doc)
        results = check(oracle, doc, tuples=t)
        ru, au = walk_records(reg("untyped"), doc, t)
        rt, at = walk_records(reg(), doc, t)
        assert ru.tobytes() == rt.tobytes() and au.tobytes() == at.tobytes()
        assert all(r[0] == "ok" for r in results)
        n_ok += len(results)
    assert n_ok > 1000


# ---- on the GPU ---------------------------------------------------------------------------------------------------------
def _device_batch(docs):
    import torch
    import operator_builder_b200 as ob
    data = np.frombuffer(b"".join(docs), dtype=np.uint8)
    off = np.zeros(len(docs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    sc = ob.Scanner(0)
    res = sc.lex_batch(data, off)
    dev = torch.device("cuda:0")
    d = dict(bytes=torch.from_numpy(np.concatenate([data, np.zeros(16, np.uint8)])).to(dev), off=torch.from_numpy(off.astype(np.int64)).to(dev),
             tup=torch.from_numpy(res.tuples.view(np.int64).copy()).to(dev), toff=torch.from_numpy(res.doc_tuple_off.view(np.int64).copy()).to(dev))
    return sc, res, d


def _parse_on_device(sc, d, r, ndocs, doc_base, res_cap, arg_cap, slack=64):
    import torch
    dev = torch.device("cuda:0")
    d_res = torch.full(((res_cap + slack) * 32,), 0xAB, dtype=torch.uint8, device=dev)
    d_args = torch.full(((arg_cap + slack) * 16,), 0xAB, dtype=torch.uint8, device=dev)
    d_roff = torch.zeros(ndocs + 1, dtype=torch.int64, device=dev)
    d_tot = torch.zeros(2, dtype=torch.int64, device=dev)
    sc.parse_batch_device(r, d["bytes"].data_ptr(), d["off"].data_ptr(), ndocs, doc_base, d["tup"].data_ptr(), d["toff"].data_ptr(), d_res.data_ptr(),
                          res_cap, d_args.data_ptr(), arg_cap, d_roff.data_ptr(), d_tot.data_ptr(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return d_res.cpu().numpy(), d_args.cpu().numpy(), d_roff.cpu().numpy(), [int(x) for x in d_tot.cpu().tolist()]


def _gpu_docs():
    import operator_builder_b200 as ob
    rng = random.Random(913)
    docs = [d for _p, d in cu.fixtures()] + list(cu.TARGETED) + [typing_fuzz_doc(rng) for _ in range(1500)] + [cu.fuzz_doc_valid(rng) for _ in range(200)]
    for marker, args in ARG_TYPES.items():
        for arg in args:
            docs += [b"# " + marker + b":" + PREFIX[marker] + arg + form + b"\n" for form, _v in FORMS]
    docs += [b"# +operator-builder:field:name=a,type=int\n# +operator-builder:field:name=1,type=int\n# +operator-builder:field:name=c,type=int\n",
             b"+operator-builder:field:name=a,type=int,name=b,type=bool,name=c\n", b"+operator-builder:field:description=d\n"]
    data0, _ = ob.generate_corpus_host(200, 4096, flavour=0)
    docs += [data0.tobytes()[i * 4096:(i + 1) * 4096] for i in range(200)]
    return docs


@pytest.mark.gpu
def test_typed_kernel_matches_host_walk_and_oracle(oracle):
    """k_parse_docs<., true>: records byte-equal to the host run of the same walk; formatted == obm_parse_doc == the oracle.
    The batch mixes OBM_R_HOST documents (fixtures with in-band warnings) with typed failures."""
    import operator_builder_b200 as ob
    from tests import typed_parser_oracle as po
    docs = _gpu_docs()
    sc, res, d = _device_batch(docs)
    for kind in ("typed", "mixed"):
        r = reg(kind)
        R_, A_, roff, (nres, nargs) = _parse_on_device(sc, d, r, len(docs), 7000, 10 ** 6, 10 ** 6)
        Rr = R_[:nres * 32].view(RES_DT); Aa = A_[:nargs * 16].view(ARG_DT)
        arg_at, seen = 0, {"host": 0, "err": 0, "panic": 0, "missing": 0}
        for i, doc in enumerate(docs):
            t = res.tuples[int(res.doc_tuple_off[i]):int(res.doc_tuple_off[i + 1])]
            hr, ha = walk_records(r, doc, t, i + 7000)
            dr = Rr[int(roff[i]):int(roff[i + 1])].copy()
            assert len(dr) == len(hr), (i, doc)
            dr_rel = dr.copy()
            local = (dr_rel["flags"] & R_HOST) == 0  # OBM_R_HOST records carry arg_base 0, not a slot
            dr_rel["arg_base"][local] -= arg_at
            assert dr_rel.tobytes() == hr.tobytes(), (i, doc, dr.tolist(), hr.tolist())
            assert Aa[arg_at:arg_at + len(ha)].tobytes() == ha.tobytes(), (i, doc)
            arg_at += len(ha)
            got = format_records(r, doc, t, dr, Aa)
            assert got == ob.parse_doc_raw(r, doc, t) == po.serialize(po.parse(oracle.lex(doc), spec(kind))), (i, doc)
            fl = int(dr[-1]["flags"]) if len(dr) else 0
            seen["host"] += int(fl & R_HOST != 0); seen["err"] += int(fl & R_ERR_SETARG != 0)
            seen["panic"] += int(fl & R_PANIC != 0); seen["missing"] += int(fl & R_ERR_MISSING != 0)
        assert arg_at == nargs and nres == int(roff[-1])
        assert min(seen.values()) > 0, seen
    sc.close()


@pytest.mark.gpu
def test_typed_kernel_capacities(oracle):
    """capacities below the totals and a non-zero doc_base: the totals stay whole, nothing is written past either capacity,
    and what fits is what the full run wrote"""
    docs = _gpu_docs()
    sc, res, d = _device_batch(docs)
    r = reg()
    R0, A0, roff0, (nres, nargs) = _parse_on_device(sc, d, r, len(docs), 123, 10 ** 6, 10 ** 6)
    for rc, ac in ((nres // 2, nargs // 3), (nres - 1, nargs - 1), (0, 5)):
        R1, A1, roff1, tot = _parse_on_device(sc, d, r, len(docs), 123, rc, ac)
        assert tot == [nres, nargs] and (roff1 == roff0).all()
        assert (R1[rc * 32:] == 0xAB).all() and (A1[ac * 16:] == 0xAB).all()
        assert R1[:rc * 32].tobytes() == R0[:rc * 32].tobytes()
        # arguments: a document whose slots straddle the capacity may have written transient records it later gave back, but
        # every slot of a result that fits whole is final
        Rr = R1[:rc * 32].view(RES_DT)
        for x in Rr:
            lo, hi = int(x["arg_base"]), int(x["arg_base"]) + int(x["nargs"])
            if hi <= ac and not int(x["flags"]) & R_HOST:
                assert A1[lo * 16:hi * 16].tobytes() == A0[lo * 16:hi * 16].tobytes()
    sc.close()


@pytest.mark.gpu
def test_typed_equals_untyped_on_c4():
    """C4 at full size (2,621,440 x 4 KiB, generated on the device): the typed walk writes exactly the untyped walk's records"""
    import torch
    import operator_builder_b200 as ob
    ndocs, doc_bytes = int(os.environ.get("OBM_C4_DOCS", 2621440)), 4096
    dev = torch.device("cuda:0")
    sc = ob.Scanner(0)
    st = torch.cuda.current_stream().cuda_stream
    n = ndocs * doc_bytes
    cap = n // 16
    d_bytes = torch.empty(n, dtype=torch.uint8, device=dev)
    d_off = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
    sc.generate_corpus_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, doc_bytes, 0, 0, st)
    d_tup = torch.empty(cap, dtype=torch.int64, device=dev)
    d_toff = torch.empty(ndocs + 1, dtype=torch.int64, device=dev)
    d_status = torch.zeros(4, dtype=torch.int32, device=dev)
    sc.lex_batch_device(d_bytes.data_ptr(), d_off.data_ptr(), ndocs, n, d_tup.data_ptr(), cap, d_toff.data_ptr(), d_status.data_ptr(), None, st)
    del d_status
    out = {}
    for kind in ("untyped", "typed"):
        res_cap, arg_cap = ndocs * 12, ndocs * 48
        o = dict(res=torch.zeros(res_cap * 32, dtype=torch.uint8, device=dev), args=torch.zeros(arg_cap * 16, dtype=torch.uint8, device=dev),
                 roff=torch.zeros(ndocs + 1, dtype=torch.int64, device=dev), tot=torch.zeros(2, dtype=torch.int64, device=dev))
        sc.parse_batch_device(reg(kind), d_bytes.data_ptr(), d_off.data_ptr(), ndocs, 0, d_tup.data_ptr(), d_toff.data_ptr(), o["res"].data_ptr(),
                              res_cap, o["args"].data_ptr(), arg_cap, o["roff"].data_ptr(), o["tot"].data_ptr(), st)
        out[kind] = o
    torch.cuda.synchronize()
    U, T = out["untyped"], out["typed"]
    nres, nargs = [int(x) for x in U["tot"].tolist()]
    assert nres > ndocs and torch.equal(U["tot"], T["tot"]) and torch.equal(U["roff"], T["roff"])
    assert torch.equal(U["res"][:nres * 32], T["res"][:nres * 32]) and torch.equal(U["args"][:nargs * 16], T["args"][:nargs * 16])
    sc.close()
