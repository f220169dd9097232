#!/usr/bin/env python3
"""Transcribe the reference's FieldType vectors into tests/golden/field_types.json.

Source: internal/workload/v1/markers/field_types_internal_test.go:12-93 of the reference tree (TestFieldType_UnmarshalMarkerArg:
6 table cases, each `args{in: "<input>"}` -> wantErr).  Run where the reference tree is present; the JSON output is committed
(tests/test_marker_typing.py reads it)."""
import json
import os
import re
import sys

REF = os.environ.get("OBM_REFERENCE", "/root/reference") + "/internal/workload/v1/markers/field_types_internal_test.go"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    src = open(REF).read()
    body = src[src.index("func TestFieldType_UnmarshalMarkerArg"):src.index("func TestFieldType_String")]
    cases = [{"name": m.group(1), "in": m.group(2), "wantErr": m.group(3) == "true"}
             for m in re.finditer(r'name:\s*"([^"]*)",.*?in:\s*"([^"]*)",.*?wantErr:\s*(true|false)', body, re.S)]
    if len(cases) != 6:
        sys.exit(f"expected 6 cases, found {len(cases)}")
    out = {"source": "internal/workload/v1/markers/field_types_internal_test.go:12-93", "cases": cases}
    with open(os.path.join(ROOT, "tests", "golden", "field_types.json"), "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
