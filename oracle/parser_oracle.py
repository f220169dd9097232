"""CPU ORACLE (test infrastructure) for the lexer's only consumer: a pure-Python restatement of
/root/reference/internal/markers/parser/{parser,peek,position,consumed,state,definition,emit,error}.go
@ 2827f233, fed with the lexeme stream of oracle/lexer_oracle.c.

PARITY UNPINNED: the reference has no parser tests (SURVEY.md section 4); this follows the source.
Modelled: which lexemes are consumed, scopeBuffer / MarkerText, registry lookup (definition.go:13-21),
LookupArgument filtering, value typing through strconv (state.go:95-153), error results (error.go:8-22).
NOT modelled (needs the Go struct types behind marker.Define): Argument.SetValue type conversion errors
(marker/argument.go:91-127) and InflateObject's missing-argument check (marker/marker.go:65-95) -- every
SetArgument is taken to succeed and emit() always succeeds.
"""
import struct
from decimal import Decimal

(ERROR, COMMENT, MARKER_START, SCOPE, SEPARATOR, ARG, ARG_ASSIGNMENT, ARG_DELIMITER, STRING, FLOAT, INTEGER, SYNTHETIC_BOOL,
 BOOL, QUOTE) = range(14)
MARKER_END, WARNING, EOF = 18, 19, 20

ZERO = (ERROR, b"", 0, 0)  # receive from the closed channel: lexer.go:51-53

PARSE_BOOL_TRUE = {b"1", b"t", b"T", b"TRUE", b"true", b"True"}
PARSE_BOOL_FALSE = {b"0", b"f", b"F", b"FALSE", b"false", b"False"}
F32_OVERFLOW = 2 ** 128 - 2 ** 103  # smallest magnitude that rounds to +Inf in float32
F32_OVERFLOW_DEC = Decimal(F32_OVERFLOW)


def read_float_magnitude(v: bytes) -> Decimal:
    """|value| of a decimal literal as strconv's readFloat (atof.go) reads it, exactly: sign, digits with one '.', then
    an exponent whose digits stop accumulating once it reaches 10000 (so "1e100000" reads as 1e10000).  The digit
    string goes into a Decimal as it is: no int() (4,300-digit limit) and no float() (inexact, inf)."""
    i, n = 0, len(v)
    if i < n and v[i] in b"+-":
        i += 1
    digits = bytearray()
    sawdot, dp = False, 0
    while i < n:
        c = v[i]
        if c == 0x2E:  # '.'
            if sawdot:
                break
            sawdot, dp = True, len(digits)
        elif 0x30 <= c <= 0x39:
            if c == 0x30 and not digits:  # leading zeros
                dp -= 1
            else:
                digits.append(c)
        else:
            break
        i += 1
    if not sawdot:
        dp = len(digits)
    if i < n and v[i] in b"eE":
        i += 1
        esign = 1
        if i < n and v[i] in b"+-":
            esign = -1 if v[i] == 0x2D else 1
            i += 1
        e = 0
        while i < n and 0x30 <= v[i] <= 0x39:
            if e < 10000:
                e = e * 10 + v[i] - 0x30
            i += 1
        dp += esign * e
    if not digits:
        return Decimal(0)
    return Decimal(f"{digits.decode()}E{dp - len(digits)}")  # 0.d1d2... * 10**dp


def go_quote(b: bytes) -> str:
    """strconv.Quote: the lexer oracle's (lexer_oracle.c go_quote, Unicode 13.0 IsPrint), so that both oracles quote alike.
    Values reach it with white space of any kind (consumedWhitespaced takes Unicode white space into a bool literal) and
    with any text (a FieldType value)."""
    from oracle import quote
    return quote(b).decode("utf-8")


class Parser:
    def __init__(self, lexemes, registry):
        """lexemes: list of (type, value bytes, line, col); registry: {marker name bytes: set(arg name bytes)}"""
        self.lx = list(lexemes)
        self.i = 0
        self.registry = registry
        self.scope_buffer = b""
        self.peek_stack = [ZERO, ZERO, ZERO]
        self.peek_count = 0
        self.current = (ERROR, b"", 0, 0)
        self.definition = None  # (name, argset)
        self.results = []
        self.loaded = []  # names for which loadDefinition succeeded, in order (definition.go:13-21)

    # lexer.NextLexeme on a channel that is closed after the last lexeme
    def _next_lexeme(self):
        if self.i < len(self.lx):
            v = self.lx[self.i]
            self.i += 1
            return v
        return ZERO

    # peek.go:8-22
    def peek(self):
        if self.peek_count > 0:
            return self.peek_stack[self.peek_count - 1]
        self.peek_count = 1
        self.peek_stack[2] = self.peek_stack[1]
        self.peek_stack[1] = self.peek_stack[0]
        self.peek_stack[0] = self._next_lexeme()
        return self.peek_stack[0]

    def peeked(self, t):
        return self.peek()[0] == t

    # position.go:7-20
    def next(self):
        if self.peek_count > 0:
            self.peek_count -= 1
        else:
            self.peek_stack[2] = self.peek_stack[1]
            self.peek_stack[1] = self.peek_stack[0]
            self.peek_stack[0] = self._next_lexeme()
        self.scope_buffer += self.peek_stack[self.peek_count][1]
        self.current = self.peek_stack[self.peek_count]

    # position.go:23-31
    def discard(self):
        if self.peek_count > 1:
            for k in range(self.peek_count, 0, -1):
                if k < 3:
                    self.peek_stack[k] = self.peek_stack[k - 1]
        self.peek_stack[0] = self._next_lexeme()

    def flush(self):
        self.scope_buffer = b""
        self.definition = None

    # consumed.go:8-16
    def consumed(self, t):
        if self.peek()[0] == t:
            self.next()
            return True
        return False

    # error.go:8-22
    def error(self, msg: str):
        name = self.definition[0].decode() if self.definition else "Unknown Marker"
        _t, _v, line, col = self.current
        self.results.append(("error", f"{msg}, on marker {name} at {{line:{line} column:{col}}}", self.scope_buffer))
        return None

    # emit.go:8-24 (InflateObject taken to succeed)
    def emit(self):
        self.results.append(("ok", self.definition[0], self.scope_buffer, self.args))
        self.flush()

    # ---- state.go ----
    def run(self):
        state = self.start_parse
        while state is not None:
            state = state()
        return self.results

    def start_parse(self):  # state.go:13-27
        if self.peeked(COMMENT):
            self.discard()
            return self.parse
        if self.consumed(MARKER_START):
            return self.parse_marker_start
        if self.consumed(EOF):
            return None
        return self.parse

    def parse(self):  # state.go:29-46
        if self.peeked(COMMENT):
            self.discard()
            return self.parse
        if self.consumed(MARKER_START):
            return self.parse_marker_start
        if self.consumed(EOF):
            return None
        if self.consumed(ERROR):
            return self.error(self.current[1].decode("utf-8", "replace"))
        self.next()
        self.scope_buffer = b""
        return self.parse

    def parse_marker_start(self):  # :48-54
        return self.parse_scope if self.consumed(SCOPE) else self.parse

    def parse_scope(self):  # :56-62
        return self.parse_separator if self.consumed(SEPARATOR) else self.parse

    def parse_separator(self):  # :64-77
        if self.consumed(SCOPE):
            return self.parse_scope
        if self.peeked(ARG):
            name = self.scope_buffer[:-1]  # definition.go:14: strip the trailing ':'
            if name in self.registry:
                self.definition = (name, self.registry[name])
                self.loaded.append(name)
                self.args = []
                return self.parse_arg
        self.flush()
        return self.parse

    def parse_arg(self):  # :79-93
        if self.consumed(ARG):
            if self.current[1] in self.definition[1]:
                arg = self.current[1]
                if self.peeked(ARG_ASSIGNMENT):
                    self.next()
                return self.parse_arg_value(arg)
        return self.parse

    def strip_quotes(self):  # :171-175
        if self.peeked(QUOTE):
            self.next()

    def parse_arg_value(self, arg):  # :95-153
        self.strip_quotes()
        if self.peeked(SYNTHETIC_BOOL):
            v = self.peek()[1]
            b = self._parse_bool(v)
            if b is None:
                return self.error(f'strconv.ParseBool: parsing {go_quote(v)}: invalid syntax')
            self.args.append((arg, "bool", v))
            self.discard()
        elif self.consumed(BOOL):
            v = self.current[1]
            if self._parse_bool(v) is None:
                return self.error(f'strconv.ParseBool: parsing {go_quote(v)}: invalid syntax')
            self.args.append((arg, "bool", v))
        elif self.consumed(INTEGER):
            self.args.append((arg, "int", self.current[1]))  # the lexer already validated strconv.Atoi (state.go:269)
        elif self.consumed(FLOAT):
            v = self.current[1]
            if read_float_magnitude(v) >= F32_OVERFLOW_DEC:
                return self.error(f'strconv.ParseFloat: parsing {go_quote(v)}: value out of range')
            self.args.append((arg, "float", v))
        elif self.consumed(STRING):
            self.args.append((arg, "string", self.current[1]))
            self.strip_quotes()
        else:
            return self.parse
        return self.parse_more_args

    def parse_more_args(self):  # :155-169
        if self.consumed(ARG_DELIMITER):
            return self.parse_arg
        if self.consumed(MARKER_END):
            self.emit()
            return self.parse
        return self.parse

    @staticmethod
    def _parse_bool(v):
        if v in PARSE_BOOL_TRUE:
            return True
        if v in PARSE_BOOL_FALSE:
            return False
        return None


def parse(lexemes, registry):
    return Parser(lexemes, registry).run()


def serialize(results) -> bytes:
    """Same record format as obm_parse_doc (csrc/obm_parse.cpp)."""
    out = bytearray()
    for r in results:
        if r[0] == "error":
            msg = r[1].encode("utf-8", "replace")
            out += struct.pack("<BI", 1, len(msg)) + msg + struct.pack("<I", len(r[2])) + r[2]
        else:
            _ok, name, text, args = r
            out += struct.pack("<BI", 0, len(name)) + name + struct.pack("<I", len(text)) + text + struct.pack("<I", len(args))
            for a, kind, v in args:
                k = {"bool": 0, "int": 1, "float": 2, "string": 3}[kind]
                out += struct.pack("<I", len(a)) + a + struct.pack("<BI", k, len(v)) + v
    return bytes(out)


# the three markers operator-builder registers (internal/workload/v1/markers/field_marker.go:19,26-38,
# collection_field_marker.go:13,22, resource_marker.go:25,47-57); argument names are lowerCamelCase field names
OPERATOR_BUILDER_REGISTRY = {
    b"+operator-builder:field": {b"name", b"type", b"description", b"default", b"replace"},
    b"+operator-builder:collection:field": {b"name", b"type", b"description", b"default", b"replace"},
    b"+operator-builder:resource": {b"field", b"collectionField", b"value", b"include"},
}
