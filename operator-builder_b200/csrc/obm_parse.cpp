/*
 * obm_parse.cpp -- host-side mirror of the lexer's only consumer, internal/markers/parser, running on
 * the GPU tuple stream (through obm_stream_*): SURVEY.md section 8(f) rank 1, the parser token contract
 * of 8(a) a17.
 *
 * Follows parser/{parser,peek,position,consumed,state,definition,emit,error}.go @ 2827f233 state by state:
 *   startParse/parse        state.go:13-46     parseMarkerStart/Scope/Separator   state.go:48-77
 *   parseArg                state.go:79-93     parseArgValue                      state.go:95-153
 *   parseMoreArgs           state.go:155-169   stripQuotes                        state.go:171-175
 *   scopeBuffer/MarkerText  position.go:18, emit.go:8-24      error results       error.go:8-22
 *   registry lookup         definition.go:13-21 (name = scopeBuffer minus the trailing ':')
 * Definitions added with their Go struct types (obm_registry_define) also get what marker.Define builds from them:
 *   Argument.SetValue       marker/argument.go:91-127 via Definition.SetArgument marker/marker.go:53-63
 *   InflateObject           marker/marker.go:65-95 (missing required arguments), run by emit.go:8-24
 * Definitions added with names only (obm_registry_add) keep the untyped semantics: every SetArgument succeeds and emit()
 * always succeeds.  Unpinned (no Go toolchain ran them): the %v / %q texts of the messages, restated from fmt and
 * strconv; the order of InflateObject's missing-argument list (Go iterates a map; here definition order).
 *
 * Output records (little endian), one per Result, in order:
 *   ok     [u8 0][u32 nlen][marker name][u32 tlen][MarkerText][u32 nargs] { [u32 alen][arg][u8 kind][u32 vlen][value] }
 *          typed definitions then add the inflated object, per definition field in order:
 *          [u32 nfields] { [u32 flen][field][u8 set] (set: [u8 kind][u32 vlen][value] of the field's last writer) }
 *   error  [u8 1][u32 mlen][message][u32 tlen][MarkerText]            (an error ends the document, parser.go:63-73)
 *   panic  [u8 2][u32 mlen][message][u32 tlen][MarkerText]            (reflect.Set panics on the parser goroutine: the
 *                                                                      reference process dies; nothing follows it)
 * kind: 0 bool, 1 int, 2 float, 3 string.
 */
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/obmarkers.h"
#include "go_unicode_tables.h"
#include "obm_core.h"
#include "obm_parse_dev.h"

struct obm_registry {
    struct Def { std::string name; std::vector<std::string> args; std::vector<uint8_t> types; /* empty: untyped */ };
    std::vector<Def> defs;
    bool typed() const { for (const auto &d : defs) if (!d.types.empty()) return true; return false; }
};

extern "C" obm_registry *obm_registry_new(void) { return new (std::nothrow) obm_registry(); }
extern "C" void obm_registry_free(obm_registry *r) { delete r; }
extern "C" int obm_registry_add(obm_registry *r, const char *marker_name, const char *const *arg_names, uint32_t nargs) {
    if (!r || !marker_name) return OBM_E_ARG;
    obm_registry::Def d; d.name = marker_name;
    for (uint32_t i = 0; i < nargs; i++) d.args.push_back(arg_names[i]);
    r->defs.push_back(d);
    return OBM_OK;
}
/* The three markers operator-builder registers: internal/workload/v1/markers/field_marker.go:19,26-38,
 * collection_field_marker.go:13,22, resource_marker.go:25,47-57 (argument names = lowerCamelCase field names). */
extern "C" obm_registry *obm_registry_operator_builder(void) {
    obm_registry *r = obm_registry_new();
    if (!r) return nullptr;
    const char *field[] = {"name", "type", "description", "default", "replace"};
    const char *res[] = {"field", "collectionField", "value", "include"};
    obm_registry_add(r, "+operator-builder:field", field, 5);
    obm_registry_add(r, "+operator-builder:collection:field", field, 5);
    obm_registry_add(r, "+operator-builder:resource", res, 4);
    return r;
}

/* marker.Define(name, T{}) of the three markers (internal/workload/v1/markers/markers.go:20-25, :92-113): the arguments are
 * T's exported fields, named lowerCamelCase (argument.go:46-89); pointers and `marker:",optional"` fields are optional.
 *   FieldMarker / CollectionFieldMarker  field_marker.go:26-38: Name string, Type FieldType, Description *string,
 *                                        Default interface{} `marker:",optional"`, Replace *string
 *   ResourceMarker                       resource_marker.go:47-57: Field *string, CollectionField *string, Value interface{},
 *                                        Include *bool */
extern "C" int obm_registry_define(obm_registry *r, int marker_type) {
    using namespace obmr;
    if (!r) return OBM_E_ARG;
    obm_registry::Def d;
    const uint8_t RQ = TY_REQUIRED;
    if (marker_type == OBM_FIELD_MARKER || marker_type == OBM_COLLECTION_MARKER) {
        d.name = marker_type == OBM_FIELD_MARKER ? "+operator-builder:field" : "+operator-builder:collection:field";
        d.args = {"name", "type", "description", "default", "replace"};
        d.types = {(uint8_t)(TY_STRING | RQ), (uint8_t)(TY_FIELDTYPE | RQ), TY_STRING, TY_ANY, TY_STRING};
    } else if (marker_type == OBM_RESOURCE_MARKER) {
        d.name = "+operator-builder:resource";
        d.args = {"field", "collectionField", "value", "include"};
        d.types = {TY_STRING, TY_STRING, (uint8_t)(TY_ANY | RQ), TY_BOOL};
    } else return OBM_E_ARG;
    if (d.args.size() > obmr::TY_MAX_FIELDS) return OBM_E_ARG; /* what TypedSink tracks */
    for (auto &x : r->defs) if (x.name == d.name) { x = d; return OBM_OK; } /* Registry.Add replaces by name (registry.go:20-22) */
    r->defs.push_back(d);
    return OBM_OK;
}

/* names of the registry (internal use by the device index, obm_lib.cu) */
extern "C" uint32_t obm_registry_names(const obm_registry *r, const char **names, uint32_t *lens, uint32_t cap) {
    if (cap == 0xFFFFFFFFu) return (uint32_t)r->defs.size(); /* count only */
    uint32_t n = 0;
    for (const auto &d : r->defs) { if (n >= cap) break; names[n] = d.name.data(); lens[n] = (uint32_t)d.name.size(); n++; }
    return n;
}

namespace {

struct Lx { int32_t type; std::string value; int64_t line, col; };

void put_u32(std::string &o, uint32_t v) { o.append((const char *)&v, 4); }

/* strconv.Quote of the byte strings that can reach a strconv error here */
std::string go_quote_simple(const std::string &s) {
    static const char hex[] = "0123456789abcdef";
    std::string o = "\"";
    for (unsigned char c : s) {
        if (c == '"' || c == '\\') { o.push_back('\\'); o.push_back((char)c); }
        else if (c == '\n') o += "\\n"; else if (c == '\t') o += "\\t"; else if (c == '\r') o += "\\r";
        else if (c == '\v') o += "\\v"; else if (c == '\f') o += "\\f";
        else if (c < 0x20) { o += "\\x"; o.push_back(hex[c >> 4]); o.push_back(hex[c & 15]); }
        else if (c == 0x7F) o += "\\u007f";
        else o.push_back((char)c);
    }
    o.push_back('"');
    return o;
}

bool parse_bool_ok(const std::string &v) { /* strconv.ParseBool */
    static const char *ok[] = {"1", "t", "T", "TRUE", "true", "True", "0", "f", "F", "FALSE", "false", "False"};
    for (const char *k : ok) if (v == k) return true;
    return false;
}

/* does the (lexer-validated) decimal literal overflow float32?  value >= 2^128 - 2^103 = 3.4028235677973366e38 */
bool float32_overflows(const std::string &v) {
    static const char *T = "340282356779733661637539395458142568448"; /* 2^128 - 2^103, 39 digits */
    size_t i = 0;
    if (i < v.size() && (v[i] == '+' || v[i] == '-')) i++;
    std::string digits; long long dp = 0; bool dot = false, any = false;
    for (; i < v.size(); i++) {
        char c = v[i];
        if (c == '.') { dot = true; continue; }
        if (c < '0' || c > '9') break;
        if (digits.empty() && c == '0') { if (dot) dp--; continue; }
        digits.push_back(c); any = true;
        if (!dot) dp++;
    }
    if (!any) return false;
    if (i < v.size() && (v[i] == 'e' || v[i] == 'E')) {
        i++; int sg = 1; long long e = 0;
        if (i < v.size() && (v[i] == '+' || v[i] == '-')) { if (v[i] == '-') sg = -1; i++; }
        for (; i < v.size() && v[i] >= '0' && v[i] <= '9'; i++) if (e < 10000) e = e * 10 + (v[i] - '0');
        dp += sg * e;
    }
    /* value = 0.d1d2... * 10^dp */
    if (dp > 39) return true;
    if (dp < 39) return false;
    for (size_t k = 0; k < 39; k++) {
        char c = k < digits.size() ? digits[k] : '0';
        if (c > T[k]) return true;
        if (c < T[k]) return false;
    }
    return true;
}

/* ---- SetArgument / InflateObject messages (marker/argument.go:91-127, marker.go:53-95) ---- */

/* %v of the Go value strconv produced from the lexeme (state.go:95-153) */
std::string go_v_int(const std::string &v) { return std::to_string(strtoll(v.c_str(), nullptr, 10)); } /* Atoi: "007" -> 7, "-0" -> 0 */
std::string go_v_bool(const std::string &v) { return (v == "1" || v == "t" || v == "T" || v == "TRUE" || v == "true" || v == "True") ? "true" : "false"; }
/* ParseFloat(v, 32) widened to float64, printed by %v: strconv.FormatFloat(f, 'g', -1, 64) -- the shortest decimal that
 * reads back as f, in %e form when its exponent is < -4 or >= 6 (ftoa.go: eprec = 6 for the shortest 'g') */
std::string go_v_float32(const std::string &v) {
    const double f = (double)strtof(v.c_str(), nullptr); /* correctly rounded to float32 */
    const bool neg = std::signbit(f);
    std::string o = neg ? "-" : "";
    if (f == 0) return o + "0";
    const double af = neg ? -f : f;
    /* shortest p digits: the correctly rounded p-digit decimal, or a neighbour of it when af is a power of two (its rounding
     * interval is narrower below than above); among p-digit decimals that read back as af, the closest */
    std::string digs; int e10 = 0;
    for (int p = 1; p <= 17 && digs.empty(); p++) {
        char buf[64];
        snprintf(buf, sizeof buf, "%.*e", p - 1, af);
        std::string m0; const char *e = strchr(buf, 'e');
        for (const char *c = buf; c < e; c++) if (*c != '.') m0.push_back(*c);
        const int x0 = atoi(e + 1) - (p - 1);
        const unsigned long long M = strtoull(m0.c_str(), nullptr, 10);
        long double best = -1;
        for (const unsigned long long cand : {M, M - 1, M + 1}) {
            if (cand == 0) continue;
            snprintf(buf, sizeof buf, "%llue%d", cand, x0);
            if (strtod(buf, nullptr) != af) continue;
            const long double d = fabsl(strtold(buf, nullptr) - (long double)af);
            if (best >= 0 && d >= best) continue;
            best = d; digs = std::to_string(cand); e10 = x0 + (int)digs.size() - 1;
        }
    }
    while (digs.size() > 1 && digs.back() == '0') digs.pop_back();
    const int nd = (int)digs.size(), dp = e10 + 1; /* value = 0.d1d2... * 10^dp */
    const int x = dp - 1;
    if (x < -4 || x >= 6) {
        o.push_back(digs[0]);
        if (nd > 1) { o.push_back('.'); o += digs.substr(1); }
        o += x < 0 ? "e-" : "e+";
        const int ax = x < 0 ? -x : x;
        if (ax < 10) o.push_back('0');
        o += std::to_string(ax);
        return o;
    }
    if (dp > 0) { for (int k = 0; k < dp; k++) o.push_back(k < nd ? digs[k] : '0'); } else o.push_back('0');
    if (nd > dp) { o.push_back('.'); for (int k = dp; k < nd; k++) o.push_back(k < 0 ? '0' : digs[k]); }
    return o;
}
const char *go_type_name(uint32_t vk) { return vk == 0 ? "bool" : vk == 1 ? "int" : vk == 2 ? "float64" : "string"; }
std::string go_v(uint32_t vk, const std::string &v) { return vk == 0 ? go_v_bool(v) : vk == 1 ? go_v_int(v) : vk == 2 ? go_v_float32(v) : v; }
/* the error of SetArgument(arg, value) for an argument of type ty (obmr::setarg_outcome says it failed); "" = panic */
std::string setarg_message(uint8_t ty, uint32_t vk, const std::string &v, const std::string &arg) {
    std::string m;
    switch (ty & obmr::TY_KIND) {
    case obmr::TY_FIELDTYPE:
        if (vk == 3) m = "unable to unmarshal arg value " + go_quote_simple(v) + ", unable to parse field, " + v + " into FieldType";
        else m = "unable to unmarshal arg value, cannot convert " + go_v(vk, v) + " to string";
        break;
    default: /* string / *string / *bool: "%q" of reflect.Type (the element type for pointers) */
        m = std::string("incorrect type, wanted \"") + ((ty & obmr::TY_KIND) == obmr::TY_BOOL ? "bool" : "string") + "\" but received \"" + go_type_name(vk) + "\"";
    }
    return m + " on arg " + arg;
}
std::string panic_message(uint32_t vk) { return std::string("reflect.Set: value of type ") + go_type_name(vk) + " is not assignable to type string"; }
/* InflateObject's error as emit wraps it: fmt %q of the []string of missing fields */
std::string missing_message(const obm_registry::Def &d, uint32_t mask) {
    std::string m = "unable to inflate object, missing arguments: [";
    bool first = true;
    for (size_t j = 0; j < d.args.size(); j++) if ((mask >> j) & 1u) { if (!first) m.push_back(' '); first = false; m += go_quote_simple(d.args[j]); }
    return m + "]";
}
void put_record(std::string &o, uint8_t type, const std::string &m, const std::string &text) {
    o.push_back((char)type); put_u32(o, (uint32_t)m.size()); o += m; put_u32(o, (uint32_t)text.size()); o += text;
}

struct Parser {
    obm_stream *s; const obm_registry *reg;
    std::string scope;             /* scopeBuffer */
    Lx stack[3]; int peek_count = 0;
    Lx current;
    const obm_registry::Def *def = nullptr;
    struct Arg { std::string name; uint8_t kind; std::string value; };
    std::vector<Arg> args;
    bool panicked = false;
    std::string out; int64_t nresults = 0;

    Lx next_lexeme() {
        obm_lexeme l; Lx r;
        if (obm_stream_next(s, &l)) { r.type = l.type; r.value.assign((const char *)l.value, l.value_len); r.line = l.line; r.col = l.column; }
        else { r.type = 0; r.line = r.col = 0; }
        return r;
    }
    const Lx &peek() { /* peek.go:8-22 */
        if (peek_count > 0) return stack[peek_count - 1];
        peek_count = 1; stack[2] = stack[1]; stack[1] = stack[0]; stack[0] = next_lexeme();
        return stack[0];
    }
    bool peeked(int t) { return peek().type == t; }
    void next() { /* position.go:7-20 */
        if (peek_count > 0) peek_count--; else { stack[2] = stack[1]; stack[1] = stack[0]; stack[0] = next_lexeme(); }
        scope += stack[peek_count].value; current = stack[peek_count];
    }
    void discard() { /* position.go:23-31 */
        if (peek_count > 1) for (int i = peek_count < 3 ? peek_count : 2; i > 0; i--) stack[i] = stack[i - 1];
        stack[0] = next_lexeme();
    }
    bool consumed(int t) { if (peek().type == t) { next(); return true; } return false; }
    void flush() { scope.clear(); def = nullptr; }
    void error(const std::string &msg) { /* error.go:8-22 */
        char pos[96]; snprintf(pos, sizeof pos, "{line:%lld column:%lld}", (long long)current.line, (long long)current.col);
        std::string m = msg + ", on marker " + (def ? def->name : std::string("Unknown Marker")) + " at " + pos;
        out.push_back(1); put_u32(out, (uint32_t)m.size()); out += m; put_u32(out, (uint32_t)scope.size()); out += scope;
        nresults++;
    }
    bool emit() { /* emit.go:8-24; false: InflateObject failed (the caller reports it through error()) */
        uint32_t missing = 0;
        if (!def->types.empty()) /* InflateObject, marker.go:65-95 */
            for (size_t j = 0; j < def->args.size(); j++) {
                if (!(def->types[j] & obmr::TY_REQUIRED)) continue;
                bool set = false;
                for (const Arg &a : args) set = set || a.name == def->args[j];
                if (!set) missing |= 1u << j;
            }
        if (missing) { error(missing_message(*def, missing)); return false; }
        out.push_back(0); put_u32(out, (uint32_t)def->name.size()); out += def->name; put_u32(out, (uint32_t)scope.size()); out += scope;
        put_u32(out, (uint32_t)args.size());
        for (const Arg &a : args) { put_u32(out, (uint32_t)a.name.size()); out += a.name; out.push_back((char)a.kind); put_u32(out, (uint32_t)a.value.size()); out += a.value; }
        if (!def->types.empty()) { /* the inflated object: each field's last writer (marker.go:59) */
            put_u32(out, (uint32_t)def->args.size());
            for (const std::string &f : def->args) {
                put_u32(out, (uint32_t)f.size()); out += f;
                const Arg *w = nullptr;
                for (const Arg &a : args) if (a.name == f) w = &a;
                out.push_back(w ? 1 : 0);
                if (w) { out.push_back((char)w->kind); put_u32(out, (uint32_t)w->value.size()); out += w->value; }
            }
        }
        nresults++;
        flush();
        return true;
    }
    bool lookup_arg(const std::string &n) const { for (const auto &a : def->args) if (a == n) return true; return false; }
    /* Definition.SetArgument (marker.go:53-63); false: the parse ends (an error Result, or the panic record) */
    bool set_argument(const std::string &arg, uint32_t vk, const std::string &v) {
        if (def->types.empty()) return true;
        size_t j = 0;
        while (def->args[j] != arg) j++;
        const uint32_t out_ = obmr::setarg_outcome(def->types[j], vk, (const uint8_t *)v.data(), (uint32_t)v.size());
        if (out_ == 0) return true;
        if (out_ == 2) { put_record(out, 2, panic_message(vk), scope); nresults++; panicked = true; return false; }
        error(setarg_message(def->types[j], vk, v, arg));
        return false;
    }

    enum St { S_START, S_PARSE, S_MARKER_START, S_SCOPE, S_SEPARATOR, S_ARG, S_MORE, S_STOP };
    void run() {
        St st = S_START;
        while (st != S_STOP) {
            switch (st) {
            case S_START: case S_PARSE: /* state.go:13-46 */
                if (peeked(OBM_K_COMMENT)) { discard(); st = S_PARSE; }
                else if (consumed(OBM_K_MARKER_START)) st = S_MARKER_START;
                else if (consumed(OBM_K_EOF)) st = S_STOP;
                else if (st == S_PARSE && consumed(OBM_K_ERROR)) { error(current.value); st = S_STOP; }
                else if (st == S_START) st = S_PARSE;
                else { next(); scope.clear(); st = S_PARSE; }
                break;
            case S_MARKER_START: st = consumed(OBM_K_SCOPE) ? S_SCOPE : S_PARSE; break;
            case S_SCOPE: st = consumed(OBM_K_SEPARATOR) ? S_SEPARATOR : S_PARSE; break;
            case S_SEPARATOR: /* state.go:64-77 */
                if (consumed(OBM_K_SCOPE)) { st = S_SCOPE; break; }
                if (peeked(OBM_K_ARG) && !scope.empty()) {
                    std::string name = scope.substr(0, scope.size() - 1);
                    const obm_registry::Def *d = nullptr;
                    for (const auto &x : reg->defs) if (x.name == name) { d = &x; break; }
                    if (d) { def = d; args.clear(); st = S_ARG; break; }
                }
                flush(); st = S_PARSE;
                break;
            case S_ARG: { /* state.go:79-93 + parseArgValue :95-153 */
                if (!consumed(OBM_K_ARG) || !lookup_arg(current.value)) { st = S_PARSE; break; }
                std::string arg = current.value;
                if (peeked(OBM_K_ARG_ASSIGNMENT)) next();
                if (peeked(OBM_K_QUOTE)) next();
                if (peeked(OBM_K_SYNTHETIC_BOOL)) {
                    std::string v = peek().value;
                    if (!parse_bool_ok(v)) { error("strconv.ParseBool: parsing " + go_quote_simple(v) + ": invalid syntax"); st = S_STOP; break; }
                    if (!set_argument(arg, 0, v)) { st = S_STOP; break; }
                    args.push_back(Arg{arg, 0, v}); discard();
                } else if (consumed(OBM_K_BOOL_LITERAL)) {
                    if (!parse_bool_ok(current.value)) { error("strconv.ParseBool: parsing " + go_quote_simple(current.value) + ": invalid syntax"); st = S_STOP; break; }
                    if (!set_argument(arg, 0, current.value)) { st = S_STOP; break; }
                    args.push_back(Arg{arg, 0, current.value});
                } else if (consumed(OBM_K_INTEGER_LITERAL)) {
                    if (!set_argument(arg, 1, current.value)) { st = S_STOP; break; }
                    args.push_back(Arg{arg, 1, current.value});
                } else if (consumed(OBM_K_FLOAT_LITERAL)) {
                    if (float32_overflows(current.value)) { error("strconv.ParseFloat: parsing " + go_quote_simple(current.value) + ": value out of range"); st = S_STOP; break; }
                    if (!set_argument(arg, 2, current.value)) { st = S_STOP; break; }
                    args.push_back(Arg{arg, 2, current.value});
                } else if (consumed(OBM_K_STRING_LITERAL)) {
                    if (!set_argument(arg, 3, current.value)) { st = S_STOP; break; }
                    args.push_back(Arg{arg, 3, current.value});
                    if (peeked(OBM_K_QUOTE)) next();
                } else { st = S_PARSE; break; }
                st = S_MORE;
                break;
            }
            case S_MORE: /* state.go:155-169 */
                if (consumed(OBM_K_ARG_DELIMITER)) st = S_ARG;
                else if (consumed(OBM_K_MARKER_END)) st = emit() ? S_PARSE : S_STOP;
                else st = S_PARSE;
                break;
            default: st = S_STOP;
            }
        }
    }
};

} // namespace

/* registry -> the flat form the device walk uses (csrc/obm_parse_dev.h); false when it does not fit */
extern "C" bool obm_registry_flatten(const obm_registry *r, obmr::DevTypedRegistry *D) {
    memset(D, 0, sizeof *D);
    if (r->defs.size() > 8) return false;
    uint32_t o = 0, a = 0;
    for (size_t i = 0; i < r->defs.size(); i++) {
        const auto &d = r->defs[i];
        if (o + d.name.size() > sizeof D->text) return false;
        D->name_off[i] = o; memcpy(D->text + o, d.name.data(), d.name.size()); o += (uint32_t)d.name.size();
    }
    D->name_off[r->defs.size()] = o; D->n = (uint32_t)r->defs.size();
    for (size_t i = 0; i < r->defs.size(); i++) {
        D->arg_first[i] = a;
        for (const auto &n : r->defs[i].args) {
            if (a >= 64 || o + n.size() > sizeof D->text) return false;
            D->arg_off[a++] = o; memcpy(D->text + o, n.data(), n.size()); o += (uint32_t)n.size();
        }
    }
    D->arg_first[r->defs.size()] = a; D->arg_off[a] = o;
    for (size_t i = 0; i < r->defs.size(); i++) {
        const auto &d = r->defs[i];
        if (d.types.empty()) continue;
        D->typed[i] = 1;
        for (size_t j = 0; j < d.types.size(); j++) {
            D->type[D->arg_first[i] + j] = d.types[j];
            if (d.types[j] & obmr::TY_REQUIRED) D->required[i] |= (uint8_t)(1u << j);
        }
    }
    return true;
}

/* host run of the device walk over one document (test / mirror use: the records the GPU would write) */
extern "C" int64_t obm_parse_doc_records(const obm_registry *reg, const uint8_t *doc, const obm_tuple *tuples, uint64_t ntuples, uint32_t doc_id,
                                         obm_result *res, uint64_t res_cap, obm_arg *args, uint64_t arg_cap, uint64_t *nargs_out) {
    obmr::DevTypedRegistry D;
    if (!reg || !obm_registry_flatten(reg, &D)) return OBM_E_ARG;
    obmr::TypedSink S; static_cast<obmr::Sink &>(S) = obmr::Sink{res, res_cap, args, arg_cap, 0, 0, 0, 0};
    if (reg->typed()) obmr::parse_doc<true>(D, doc, tuples, (uint32_t)ntuples, doc_id, S);
    else obmr::parse_doc<false>(static_cast<const obmr::DevRegistry &>(D), doc, tuples, (uint32_t)ntuples, doc_id, static_cast<obmr::Sink &>(S));
    if (nargs_out) *nargs_out = S.nargs;
    return S.nres;
}

extern "C" int64_t obm_results_format_doc(const obm_registry *reg, const uint8_t *doc, uint64_t doc_len, const obm_tuple *tuples, uint64_t ntuples,
                                          const obm_result *results, uint64_t nresults, const obm_arg *args_base, uint8_t **out, uint64_t *out_len) {
    if (!reg || !out || !out_len) return OBM_E_ARG;
    if (nresults == 1 && (results[0].flags & OBM_R_HOST)) return obm_parse_doc(reg, doc, doc_len, tuples, ntuples, out, out_len);
    std::string o;
    for (uint64_t i = 0; i < nresults; i++) {
        const obm_result &r = results[i];
        if (r.reg_id >= reg->defs.size()) return OBM_E_ARG;
        const obm_registry::Def &d = reg->defs[r.reg_id];
        std::string text((const char *)doc + r.text_off, r.text_len);
        if (r.flags & OBM_R_NL) text.push_back('\n');
        if (r.flags & OBM_R_OK) {
            o.push_back(0); put_u32(o, (uint32_t)d.name.size()); o += d.name; put_u32(o, (uint32_t)text.size()); o += text;
            put_u32(o, r.nargs);
            for (uint32_t a = 0; a < r.nargs; a++) {
                const obm_arg &g = args_base[r.arg_base + a];
                put_u32(o, g.name_len); o.append((const char *)doc + g.name_off, g.name_len); o.push_back((char)g.kind);
                if (g.flags & OBM_A_SYNTHETIC_TRUE) { put_u32(o, 4); o += "true"; }
                else { put_u32(o, g.val_len); o.append((const char *)doc + g.val_off, g.val_len); }
            }
            if (!d.types.empty()) { /* the inflated object: per field, the one argument not superseded */
                put_u32(o, (uint32_t)d.args.size());
                for (const std::string &f : d.args) {
                    put_u32(o, (uint32_t)f.size()); o += f;
                    const obm_arg *w = nullptr;
                    for (uint32_t a = 0; a < r.nargs; a++) {
                        const obm_arg &g = args_base[r.arg_base + a];
                        if (!(g.flags & OBM_A_SUPERSEDED) && g.name_len == f.size() && memcmp(doc + g.name_off, f.data(), f.size()) == 0) w = &g;
                    }
                    o.push_back(w ? 1 : 0);
                    if (!w) continue;
                    o.push_back((char)w->kind);
                    if (w->flags & OBM_A_SYNTHETIC_TRUE) { put_u32(o, 4); o += "true"; }
                    else { put_u32(o, w->val_len); o.append((const char *)doc + w->val_off, w->val_len); }
                }
            }
        } else if (r.flags & OBM_R_ERR_MISSING) { /* emit.go:11-13 through error.go: parser.current is the synthetic MarkerEnd */
            put_record(o, 1, missing_message(d, r.aux) + ", on marker " + d.name + " at {line:0 column:0}", text);
        } else if (r.flags & (OBM_R_ERR_SETARG | OBM_R_PANIC)) {
            const obm_arg &g = args_base[r.arg_base];
            if (g.name_len >= d.args.size() || d.types.empty()) return OBM_E_ARG;
            const std::string v = (g.flags & OBM_A_SYNTHETIC_TRUE) ? std::string("true") : std::string((const char *)doc + g.val_off, g.val_len);
            if (r.flags & OBM_R_PANIC) put_record(o, 2, panic_message(g.kind), text);
            else {
                char pos[96]; snprintf(pos, sizeof pos, "{line:%u column:%u}", g.name_off, r.aux);
                put_record(o, 1, setarg_message(d.types[g.name_len], g.kind, v, d.args[g.name_len]) + ", on marker " + d.name + " at " + pos, text);
            }
        } else { /* error.go:8-22: "<msg>, on marker <name> at {line:L column:C}" */
            const obm_arg &g = args_base[r.arg_base];
            const std::string v((const char *)doc + g.val_off, g.val_len);
            std::string m = (r.flags & OBM_R_ERR_PARSEBOOL) ? "strconv.ParseBool: parsing " + go_quote_simple(v) + ": invalid syntax"
                                                             : "strconv.ParseFloat: parsing " + go_quote_simple(v) + ": value out of range";
            char pos[96]; snprintf(pos, sizeof pos, "{line:%u column:%u}", g.name_off, r.aux);
            m += ", on marker " + d.name + " at " + pos;
            o.push_back(1); put_u32(o, (uint32_t)m.size()); o += m; put_u32(o, (uint32_t)text.size()); o += text;
        }
    }
    uint8_t *buf = (uint8_t *)malloc(o.size() ? o.size() : 1);
    if (!buf) return OBM_E_NOMEM;
    memcpy(buf, o.data(), o.size());
    *out = buf; *out_len = o.size();
    return (int64_t)nresults;
}

extern "C" int64_t obm_parse_doc(const obm_registry *reg, const uint8_t *doc, uint64_t doc_len, const obm_tuple *tuples, uint64_t ntuples,
                                 uint8_t **out, uint64_t *out_len) {
    if (!reg || !out || !out_len) return OBM_E_ARG;
    obm_stream *s = obm_stream_new(doc, doc_len, tuples, ntuples);
    if (!s) return OBM_E_NOMEM;
    Parser p; p.s = s; p.reg = reg;
    p.run();
    obm_stream_free(s);
    uint8_t *buf = (uint8_t *)malloc(p.out.size() ? p.out.size() : 1);
    if (!buf) return OBM_E_NOMEM;
    memcpy(buf, p.out.data(), p.out.size());
    *out = buf; *out_len = p.out.size();
    return p.nresults;
}
