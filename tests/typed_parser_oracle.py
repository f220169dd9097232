"""Typed marker arguments for the parser oracle (test infrastructure): oracle/parser_oracle.py's Parser extended with
Definition.SetArgument -> Argument.SetValue (internal/markers/marker/marker.go:53-63, marker/argument.go:91-127) and
InflateObject's missing-argument check (marker/marker.go:65-95), restated with the Go spec's conversion and assignability
rules, independently of the C++ code.

A registry entry given as a set of argument names (parser_oracle.OPERATOR_BUILDER_REGISTRY) keeps the untyped oracle's
semantics: every SetArgument succeeds and emit() always succeeds.  An entry given as the Go struct's fields
(OPERATOR_BUILDER_TYPED below) gets the typed ones.  Unpinned beyond the source: the fmt %v / %q texts (no Go toolchain ran
them) and the order of the missing-argument list, which Go takes from map iteration (random when two are missing; here
definition order).  Record format: csrc/obm_parse.cpp (typed OK records add the inflated object; panic records are type 2).
"""
import struct
from decimal import Decimal
from fractions import Fraction

from oracle import parser_oracle as po
from oracle.parser_oracle import (ARG, ARG_ASSIGNMENT, ARG_DELIMITER, BOOL, F32_OVERFLOW_DEC, FLOAT, INTEGER, MARKER_END,  # noqa: F401
                                  STRING, SYNTHETIC_BOOL, go_quote, read_float_magnitude)


class TypedParser(po.Parser):
    """parser_oracle.Parser with SetArgument / InflateObject for typed registry entries"""

    def parse_separator(self):  # state.go:64-77; registry.go:30-42: GetDefinition copies Fields, so each marker starts unset
        nxt = super().parse_separator()
        if nxt == self.parse_arg:
            self.fields = {}
        return nxt

    # Definition.SetArgument (marker.go:53-63) with the Go value strconv produced; False ends the parse
    def set_argument(self, arg, kind, raw, value):
        spec = self.definition[1]
        if not isinstance(spec, dict):
            return True
        try:
            err = go_set_value(spec[arg][0], kind, value)
        except GoPanic as p:  # reflect.Set panics on the parser goroutine: the process dies
            self.results.append(("panic", str(p), self.scope_buffer))
            return False
        if err is not None:
            self.error(f"{err} on arg {arg.decode()}")
            return False
        self.fields[arg] = (kind, raw)  # m.Fields[argName] = arg: the last writer wins
        return True

    def parse_arg_value(self, arg):  # state.go:95-153, SetArgument after each strconv conversion
        self.strip_quotes()
        if self.peeked(SYNTHETIC_BOOL):
            v = self.peek()[1]
            b = self._parse_bool(v)
            if b is None:
                return self.error(f'strconv.ParseBool: parsing {go_quote(v)}: invalid syntax')
            if not self.set_argument(arg, "bool", v, b):  # peeked, not consumed: parser.current is the lexeme before
                return None
            self.args.append((arg, "bool", v))
            self.discard()
        elif self.consumed(BOOL):
            v = self.current[1]
            b = self._parse_bool(v)
            if b is None:
                return self.error(f'strconv.ParseBool: parsing {go_quote(v)}: invalid syntax')
            if not self.set_argument(arg, "bool", v, b):
                return None
            self.args.append((arg, "bool", v))
        elif self.consumed(INTEGER):
            v = self.current[1]  # the lexer already validated strconv.Atoi (state.go:269)
            if not self.set_argument(arg, "int", v, int(v)):
                return None
            self.args.append((arg, "int", v))
        elif self.consumed(FLOAT):
            v = self.current[1]
            if read_float_magnitude(v) >= F32_OVERFLOW_DEC:
                return self.error(f'strconv.ParseFloat: parsing {go_quote(v)}: value out of range')
            if not self.set_argument(arg, "float", v, parse_float32(v)):
                return None
            self.args.append((arg, "float", v))
        elif self.consumed(STRING):
            v = self.current[1]
            if not self.set_argument(arg, "string", v, v):
                return None
            self.args.append((arg, "string", v))
            self.strip_quotes()
        else:
            return self.parse
        return self.parse_more_args

    def parse_more_args(self):  # state.go:155-169: an emit error ends the parse through p.error
        if self.consumed(ARG_DELIMITER):
            return self.parse_arg
        if self.consumed(MARKER_END):
            return self.parse if self.emit_typed() else None
        return self.parse

    def emit_typed(self):  # emit.go:8-24; False when InflateObject fails (the error Result is out)
        spec = self.definition[1]
        if not isinstance(spec, dict):  # names only: InflateObject taken to succeed
            self.emit()
            return True
        missing = [a for a, (gotype, optional_tag) in spec.items() if go_required(gotype, optional_tag) and a not in self.fields]
        if missing:  # marker.go:88-90 + emit.go:11-13; parser.current is the synthetic MarkerEnd
            self.error("unable to inflate object, missing arguments: [" + " ".join(go_quote(a) for a in missing) + "]")
            return False
        fields = [(a, self.fields.get(a)) for a in spec]
        self.results.append(("ok", self.definition[0], self.scope_buffer, self.args, fields))
        self.flush()
        return True


def parse(lexemes, registry):
    return TypedParser(lexemes, registry).run()


def serialize(results) -> bytes:
    """parser_oracle.serialize's record format plus panic records and the inflated object of typed OK records"""
    out = bytearray()
    kinds = {"bool": 0, "int": 1, "float": 2, "string": 3}
    for r in results:
        if r[0] == "panic":
            msg = r[1].encode("utf-8", "replace")
            out += struct.pack("<BI", 2, len(msg)) + msg + struct.pack("<I", len(r[2])) + r[2]
            continue
        out += po.serialize([r[:4]])
        if r[0] == "ok" and len(r) > 4:  # typed definition: each field's last writer
            out += struct.pack("<I", len(r[4]))
            for f, w in r[4]:
                out += struct.pack("<I", len(f)) + f + (b"\0" if w is None else struct.pack("<BBI", 1, kinds[w[0]], len(w[1])) + w[1])
    return bytes(out)


# ---- marker.Define(name, T{}) (marker/marker.go:28-123, marker/argument.go:46-89) ----
class GoPanic(Exception):
    """a run-time panic of the reference (reflect.Value.Set); the Go process aborts"""


def go_required(gotype: str, optional_tag: bool) -> bool:
    """argument.go:46-89: pointer fields and `marker:",optional"` fields are optional, every other field is required"""
    return not gotype.startswith("*") and not optional_tag


# FieldType (internal/workload/v1/markers/field_types.go:27-46): *FieldType implements parser.Unmarshaler; the names it
# accepts ("" maps to FieldUnknownType, which is an error as well)
FIELD_TYPE_NAMES = {b"string", b"int", b"bool"}
GO_VALUE_TYPE = {"bool": "bool", "int": "int", "float": "float64", "string": "string"}  # what state.go:95-153 passes


def go_convertible(v: str, t: str) -> bool:
    """The Go spec's conversion rules, for the four value types the parser passes and the targets operator-builder
    declares: identical types; any type to interface{} (it is assignable); an integer to a string type."""
    return v == t or t == "interface{}" or (v == "int" and t == "string")


def go_assignable(v: str, t: str) -> bool:
    """The Go spec's assignability: identical types, or t an interface type that v implements (interface{}: every type)"""
    return v == t or t == "interface{}"


def go_set_value(gotype: str, kind: str, value):
    """Argument.SetValue (argument.go:91-127): None on success, the error text, or GoPanic"""
    vt = GO_VALUE_TYPE[kind]
    if gotype == "FieldType":  # reflect.PtrTo(a.Type).Implements(unmarshalerType)
        if vt != "string":
            return f"unable to unmarshal arg value, cannot convert {go_v(kind, value)} to string"
        if value not in FIELD_TYPE_NAMES:
            return f"unable to unmarshal arg value {go_quote(value)}, unable to parse field, {value.decode('utf-8', 'replace')} into FieldType"
        return None
    elem = gotype[1:] if gotype.startswith("*") else gotype  # a.Pointer: a.Type.Elem()
    if not go_convertible(vt, elem):
        return f'incorrect type, wanted "{elem}" but received "{vt}"'
    if not go_assignable(vt, elem):  # reflect.Value.Set requires assignability, ConvertibleTo did not check it
        raise GoPanic(f"reflect.Set: value of type {vt} is not assignable to type {elem}")
    return None


def parse_float32(v: bytes) -> float:
    """strconv.ParseFloat(v, 32) of an in-range literal: the exact decimal rounded once to float32 (nearest, ties to even),
    widened to float64"""
    neg = v[:1] == b"-"
    q = Fraction(read_float_magnitude(v))
    if q <= Fraction(1, 2 ** 150):  # at most half the smallest subnormal: rounds to zero
        return -0.0 if neg else 0.0
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if q < Fraction(2) ** e:
        e -= 1
    scale = Fraction(2) ** (max(e, -126) - 23)  # 24-bit significand; subnormals keep the exponent of 2^-126
    m = q / scale
    n = m.numerator // m.denominator
    rem = m - n
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and n % 2 == 1):
        n += 1
    f = float(n * scale)
    return -f if neg else f


def go_format_float(x: float) -> str:
    """fmt %v of a float64 = strconv.FormatFloat(x, 'g', -1, 64): the shortest decimal that reads back as x (Python's
    repr finds the same digits), %e form when the decimal exponent is < -4 or >= 6 (ftoa.go: eprec = 6 when shortest),
    the exponent with a sign and at least two digits"""
    sign = "-" if str(x).startswith("-") else ""
    if x == 0:
        return sign + "0"
    t = Decimal(repr(abs(x))).as_tuple()
    digits = "".join(str(d) for d in t.digits)
    dp = len(digits) + t.exponent  # x = 0.d1d2... * 10**dp
    digits = digits.rstrip("0")
    exp = dp - 1
    if exp < -4 or exp >= 6:
        mant = digits[0] + ("." + digits[1:] if len(digits) > 1 else "")
        return f"{sign}{mant}e{'-' if exp < 0 else '+'}{abs(exp):02d}"
    if dp > 0:
        whole = (digits[:dp]).ljust(dp, "0")
        frac = digits[dp:]
    else:
        whole, frac = "0", "0" * (-dp) + digits
    return sign + whole + ("." + frac if frac else "")


def go_v(kind: str, value) -> str:
    """fmt %v of the Go value"""
    if kind == "bool":
        return "true" if value else "false"
    if kind == "int":
        return str(value)
    if kind == "float":
        return go_format_float(value)
    return value.decode("utf-8", "replace")


# The typed definitions operator-builder registers: {marker name: {argument name: (Go type, `marker:",optional"`)}}, the
# exported fields in declaration order, named lowerCamelCase (argument.go:46-89)
_FIELD_MARKER_T = {b"name": ("string", False), b"type": ("FieldType", False), b"description": ("*string", False),
                   b"default": ("interface{}", True), b"replace": ("*string", False)}  # field_marker.go:26-38
OPERATOR_BUILDER_TYPED = {
    b"+operator-builder:field": _FIELD_MARKER_T,
    b"+operator-builder:collection:field": dict(_FIELD_MARKER_T),  # collection_field_marker.go: the same struct
    b"+operator-builder:resource": {b"field": ("*string", False), b"collectionField": ("*string", False),
                                    b"value": ("interface{}", False), b"include": ("*bool", False)},  # resource_marker.go:47-57
}
