/*
 * obm_parse_dev.h -- the lexer's only consumer, internal/markers/parser, ON THE DEVICE (SURVEY.md 8(f) rank 1): one
 * thread per document walks the document's tuples the way parser/state.go:13-175 walks lexemes and emits compact
 * Result records instead of Go structs:
 *   registry lookup            definition.go:13-21 (marker name = scopeBuffer minus the trailing ':')
 *   known-argument filter      state.go:79-93 (LookupArgument)
 *   value typing               state.go:95-153 (ParseBool, Atoi class, ParseFloat(., 32) range)
 *   MarkerText                 position.go:18 + emit.go:8-24, as a span of the document (+ the synthetic "\n")
 *   error results              error.go:8-22 (they end the document's parse, parser.go:63-73)
 * and, for definitions added with their Go struct types (obm_registry_define; the parse_doc<true> instantiation):
 *   SetArgument                marker.go:53-63 -> argument.go:91-127 (wrong type, FieldType unmarshal, the int -> string panic)
 *   InflateObject              marker.go:65-95 (required arguments never set), run by emit.go:8-24
 *   last writer wins           marker.go:59 (Fields[argName] = arg): earlier writers of a field get OBM_A_SUPERSEDED
 * The same source is the host mirror's fast path (obm_parse.cpp: obm_results_format_doc) and is checked against
 * obm_parse_doc / oracle/parser_oracle.py in tests/test_parser_row.py.
 *
 * Scope of the device walk: documents whose tuple stream holds only plain lexemes (kinds 1..20) and LINE tuples.
 * Anything that makes a Value differ from an input slice or needs the decoder's text formatting -- PART / FLUSH /
 * DRIFT / LINEHI pseudo-tuples, in-band warnings and lexer errors -- marks the whole document OBM_R_HOST: one record,
 * and the host runs obm_parse_doc on that document's tuples (exact for everything).
 */
#ifndef OBM_PARSE_DEV_H
#define OBM_PARSE_DEV_H

#include "obm_core.h"

namespace obmr {

struct DevRegistry { /* names and argument names back to back in text[] */
    uint32_t n; uint32_t name_off[9]; uint32_t arg_first[9]; uint32_t arg_off[65]; uint8_t text[1024];
};
/* The Go type of each argument of a typed definition (obm_registry_define), appended after text[]: the untyped walk is
 * given the DevRegistry part alone, so its kernel parameter is what it was before typing existed.
 * type[a] = TY_* | TY_REQUIRED; 0 = an argument of an untyped definition (every SetArgument succeeds). */
enum : uint8_t { TY_NONE = 0, TY_STRING = 1 /* string, *string */, TY_BOOL = 2 /* *bool */, TY_FIELDTYPE = 3 /* markers.FieldType */,
                 TY_ANY = 4 /* interface{} */, TY_KIND = 7, TY_REQUIRED = 0x80 };
constexpr uint32_t TY_MAX_FIELDS = 5; /* the largest typed definition (FieldMarker) */
struct DevTypedRegistry : DevRegistry {
    uint8_t type[64];
    uint8_t required[8]; /* per definition: bit j = argument j is required (InflateObject's missingFields) */
    uint8_t typed[8];    /* per definition: 1 = added with its Go struct type */
};
/* SetArgument outcome of a value of lexeme kind vk (0 bool, 1 int, 2 float, 3 string) for an argument of type ty
 * (argument.go:91-127 with the Go spec's conversion / assignability rules): 0 ok, 1 error (OBM_R_ERR_SETARG), 2 panic */
OBM_HD uint32_t setarg_outcome(uint32_t ty, uint32_t vk, const uint8_t *v, uint32_t n) {
    switch (ty & TY_KIND) {
    case TY_STRING: return vk == 3 ? 0u : vk == 1 ? 2u : 1u; /* int is ConvertibleTo string but not assignable: reflect.Set panics */
    case TY_BOOL: return vk == 0 ? 0u : 1u;
    case TY_FIELDTYPE: /* (*FieldType).UnmarshalMarkerArg, field_types.go:27-46: "string", "int", "bool" */
        if (vk != 3) return 1u;
        if (n == 6) return (v[0] == 's' && v[1] == 't' && v[2] == 'r' && v[3] == 'i' && v[4] == 'n' && v[5] == 'g') ? 0u : 1u;
        if (n == 3) return (v[0] == 'i' && v[1] == 'n' && v[2] == 't') ? 0u : 1u;
        if (n == 4) return (v[0] == 'b' && v[1] == 'o' && v[2] == 'o' && v[3] == 'l') ? 0u : 1u;
        return 1u;
    default: return 0u; /* interface{}, untyped definitions */
    }
}

OBM_HD bool slice_eq(const uint8_t *doc, uint32_t off, uint32_t len, const uint8_t *t, uint32_t tlen) {
    if (len != tlen) return false;
    uint32_t diff = 0;
    for (uint32_t k = 0; k < len; k++) diff |= (uint32_t)doc[off + k] ^ (uint32_t)t[k]; /* independent loads: they pipeline */
    return diff == 0;
}
OBM_HD int lookup_marker(const DevRegistry &R, const uint8_t *doc, uint32_t off, uint32_t len) {
    for (uint32_t r = 0; r < R.n; r++) if (slice_eq(doc, off, len, R.text + R.name_off[r], R.name_off[r + 1] - R.name_off[r])) return (int)r;
    return -1;
}
OBM_HD bool lookup_arg(const DevRegistry &R, uint32_t def, const uint8_t *doc, uint32_t off, uint32_t len) {
    for (uint32_t a = R.arg_first[def]; a < R.arg_first[def + 1]; a++)
        if (slice_eq(doc, off, len, R.text + R.arg_off[a], R.arg_off[a + 1] - R.arg_off[a])) return true;
    return false;
}
/* strconv.ParseBool accepts exactly: 1 t T TRUE true True 0 f F FALSE false False */
OBM_HD bool parse_bool_ok(const uint8_t *v, uint32_t n) {
    if (n == 1) return v[0] == '1' || v[0] == 't' || v[0] == 'T' || v[0] == '0' || v[0] == 'f' || v[0] == 'F';
    if (n == 4) return (v[0] == 't' && v[1] == 'r' && v[2] == 'u' && v[3] == 'e') || (v[0] == 'T' && v[1] == 'R' && v[2] == 'U' && v[3] == 'E') ||
                       (v[0] == 'T' && v[1] == 'r' && v[2] == 'u' && v[3] == 'e');
    if (n == 5) return (v[0] == 'f' && v[1] == 'a' && v[2] == 'l' && v[3] == 's' && v[4] == 'e') || (v[0] == 'F' && v[1] == 'A' && v[2] == 'L' && v[3] == 'S' && v[4] == 'E') ||
                       (v[0] == 'F' && v[1] == 'a' && v[2] == 'l' && v[3] == 's' && v[4] == 'e');
    return false;
}
/* does the (lexer-validated) decimal literal overflow float32?  |value| >= 2^128 - 2^103 = 3.40282356779733661637539395458142568448e38 */
OBM_HD bool float32_overflows(const uint8_t *v, uint32_t n) {
    const char *T = "340282356779733661637539395458142568448";
    uint32_t i = 0;
    if (i < n && (v[i] == '+' || v[i] == '-')) i++;
    const uint32_t dbeg = i;
    long long dp = 0; bool dot = false, started = false; uint32_t nd = 0;
    for (; i < n; i++) {
        const uint32_t c = v[i];
        if (c == '.') { dot = true; continue; }
        if (c < '0' || c > '9') break;
        if (!started && c == '0') { if (dot) dp--; continue; }
        started = true; nd++;
        if (!dot) dp++;
    }
    const uint32_t dend = i;
    if (!started) return false;
    if (i < n && (v[i] == 'e' || v[i] == 'E')) {
        i++; int sg = 1; long long e = 0;
        if (i < n && (v[i] == '+' || v[i] == '-')) { if (v[i] == '-') sg = -1; i++; }
        for (; i < n && v[i] >= '0' && v[i] <= '9'; i++) if (e < 10000) e = e * 10 + (v[i] - '0');
        dp += sg * e;
    }
    if (dp > 39) return true;
    if (dp < 39) return false;
    uint32_t k = 0; bool st = false;
    for (uint32_t j = dbeg; j < dend && k < 39; j++) {
        const uint32_t c = v[j];
        if (c == '.') continue;
        if (!st) { if (c == '0') continue; st = true; }
        if (c > (uint32_t)T[k]) return true;
        if (c < (uint32_t)T[k]) return false;
        k++;
    }
    for (; k < 39; k++) { if ('0' > T[k]) return true; if ('0' < T[k]) return false; }
    (void)nd;
    return true;
}

/* sink: counts always, writes when the arrays are given.  res_end / arg_end: end of THIS document's slots (known from the count
 * pass): arguments of a marker that is abandoned later are written first and given back afterwards -- such transient records
 * must never land in a neighbouring document's slots (another thread writes those, in any order) */
struct Sink {
    obm_result *res; uint64_t res_end; obm_arg *args; uint64_t arg_end;
    uint64_t res_at, arg_at; /* first slot of the document (batch-global) */
    uint32_t nres, nargs;
    OBM_HD void arg(uint32_t name_off, uint32_t name_len, uint32_t kind, uint32_t val_off, uint32_t val_len, uint32_t flags) {
        if (args && arg_at + nargs < arg_end) {
            obm_arg a; a.name_off = name_off; a.val_off = val_off; a.val_len = val_len; a.name_len = (uint16_t)name_len; a.kind = (uint8_t)kind; a.flags = (uint8_t)flags;
            args[arg_at + nargs] = a;
        }
        nargs++;
    }
    OBM_HD void supersede(uint32_t slot) { /* slot: index among this document's arguments */
        if (args && arg_at + slot < arg_end) args[arg_at + slot].flags |= (uint8_t)OBM_A_SUPERSEDED;
    }
    OBM_HD void result(uint32_t doc, uint32_t tuple, uint32_t text_off, uint32_t text_len, uint32_t reg_id, uint32_t n_args, uint64_t arg_base, uint32_t flags, uint32_t aux) {
        if (res && res_at + nres < res_end) {
            obm_result r; r.doc = doc; r.tuple = tuple; r.text_off = text_off; r.text_len = text_len; r.reg_id = (uint16_t)reg_id; r.nargs = (uint16_t)n_args;
            r.arg_base = (uint32_t)arg_base; r.flags = flags; r.aux = aux;
            res[res_at + nres] = r;
        }
        nres++;
    }
};

/* the typed walk's sink also carries SetArgument / InflateObject's state of the marker being parsed (kept out of the untyped
 * walk's frame, which stays as it was) */
struct TypedSink : Sink {
    uint32_t a_idx = 0;                 /* registry index of the argument being valued */
    uint32_t set_mask = 0;              /* fields set so far (argument index in the definition) */
    uint64_t last = 0;                  /* the last writers of fields 0-3, 16 bits each: the writer's index among the marker's
                                           arguments (< 2^16 like obm_result.nargs); packed, so the walk keeps them in registers */
    uint32_t last4 = 0;                 /* and of field 4 */
};

/* 8 bytes of the document at an arbitrary offset (two aligned loads + funnel shift; the batch buffer is readable up to the
 * next 16-byte boundary behind its end, obmarkers.h) */
OBM_HD uint64_t load8(const uint8_t *p) {
    const uintptr_t a = (uintptr_t)p & ~(uintptr_t)7; const uint32_t s = (uint32_t)((uintptr_t)p & 7u) * 8u;
    const uint64_t lo = *reinterpret_cast<const uint64_t *>(a);
    if (s == 0) return lo;
    const uint64_t hi = *reinterpret_cast<const uint64_t *>(a + 8);
    return (lo >> s) | (hi << (64u - s));
}
OBM_HD bool slice_eq8(const uint8_t *doc, uint32_t off, uint32_t len, const uint8_t *t, uint32_t tlen) {
    if (len != tlen) return false;
    uint64_t diff = 0;
    uint32_t k = 0;
    for (; k + 8 <= len; k += 8) { uint64_t w = 0; for (int b = 7; b >= 0; b--) w = (w << 8) | t[k + b]; diff |= load8(doc + off + k) ^ w; }
    for (; k < len; k++) diff |= (uint64_t)((uint32_t)doc[off + k] ^ (uint32_t)t[k]);
    return diff == 0;
}

/* One document.  t: the document's slice of the tuple stream.  doc_id: what goes into the records.
 * Written as a DFA that consumes exactly ONE tuple per iteration of the outer loop (a state may hand the same tuple to
 * another state first: the parser's "peeked, not consumed" moves): a warp runs 32 documents, one per lane, and with one
 * tuple per iteration the lanes stay converged on the loop -- the walk is latency-bound on the tuple loads, which now issue
 * for all lanes at once.
 * TYPED (Reg = DevTypedRegistry, SinkT = TypedSink) adds SetArgument / InflateObject; TYPED = false (DevRegistry, Sink)
 * compiles to the walk that has no types. */
template <bool TYPED, class Reg, class SinkT>
OBM_HD void parse_doc(const Reg &R, const uint8_t *doc, const obm_tuple *t, uint32_t nt, uint32_t doc_id, SinkT &S) {
    enum St { P_PARSE, P_MSTART, P_SCOPE, P_SEP, P_ARG, P_AV1, P_AV2, P_VAL, P_VQ, P_MORE };
    uint32_t line = 1, base = 0;                                                  /* position basis (LINE tuples) */
    uint32_t sc_off = 0, sc_len = 0; bool sc_any = false, sc_nl = false, sc_broken = false; /* scopeBuffer as a span (+ "\n") */
    uint32_t cur_tuple = 0, cur_line = 0, cur_col = 0;                            /* parser.current */
    int def = -1; uint32_t marker_tuple = 0, n_args = 0; uint64_t arg_base = 0;
    uint32_t a_off = 0, a_len = 0;                                                /* the argument being valued */
    uint32_t st = P_PARSE;
    for (uint32_t i = 0; i < nt; i++) {
        const obm_tuple tu = t[i];
        const uint32_t k = OBM_TUPLE_KIND(tu), off = OBM_TUPLE_OFF(tu), len = OBM_TUPLE_LEN(tu);
        if (k == OBM_K_LINE) { base = off; line = len; continue; }
        if (k > OBM_K_EOF) { S.nres = 0; S.nargs = 0; S.result(doc_id, i, 0, 0, 0xFFFFu, 0, 0, OBM_R_HOST, k); return; } /* not modelled: obm_parse_doc decides */
        bool consumed = false, append = true, stop = false;
        for (int hop = 0; hop < 6 && !consumed; hop++) { /* at most: MSTART/SCOPE/SEP/ARG/AV1/AV2/VAL/VQ/MORE -> PARSE */
            const uint32_t was = st;
            switch (st) {
            case P_PARSE: /* state.go:13-46 */
                consumed = true;
                if (k == OBM_K_COMMENT) append = false;                              /* discard() */
                else if (k == OBM_K_MARKER_START) { marker_tuple = i; st = P_MSTART; }
                else if (k == OBM_K_EOF) stop = true;
                else { /* next(); scopeBuffer = "" */ }
                break;
            case P_MSTART: if (k == OBM_K_SCOPE) { consumed = true; st = P_SCOPE; } else st = P_PARSE; break;
            case P_SCOPE: if (k == OBM_K_SEPARATOR) { consumed = true; st = P_SEP; } else st = P_PARSE; break;
            case P_SEP: /* state.go:64-77 */
                if (k == OBM_K_SCOPE) { consumed = true; st = P_SCOPE; break; }
                st = P_PARSE;
                if (k == OBM_K_ARG && sc_any && (sc_len || sc_nl)) {
                    if (sc_broken || sc_nl) { S.nres = 0; S.nargs = 0; S.result(doc_id, i, 0, 0, 0xFFFFu, 0, 0, OBM_R_HOST, 0); return; }
                    def = -1;
                    for (uint32_t r = 0; r < R.n; r++)
                        if (slice_eq8(doc, sc_off, sc_len - 1, R.text + R.name_off[r], R.name_off[r + 1] - R.name_off[r])) { def = (int)r; break; }
                    if (def >= 0) { n_args = 0; arg_base = S.arg_at + S.nargs; st = P_ARG; if constexpr (TYPED) S.set_mask = 0; }
                }
                if (st == P_PARSE) { sc_any = false; sc_nl = false; sc_len = 0; sc_broken = false; def = -1; } /* flush() */
                break;
            case P_ARG: /* state.go:79-93 */
                if (k != OBM_K_ARG) { st = P_PARSE; break; }
                consumed = true; a_off = off; a_len = len;
                st = P_PARSE;
                for (uint32_t a = R.arg_first[def]; a < R.arg_first[def + 1]; a++)
                    if (slice_eq8(doc, off, len, R.text + R.arg_off[a], R.arg_off[a + 1] - R.arg_off[a])) { st = P_AV1; if constexpr (TYPED) S.a_idx = a; break; }
                break;
            case P_AV1: if (k == OBM_K_ARG_ASSIGNMENT) consumed = true; st = P_AV2; break;
            case P_AV2: if (k == OBM_K_QUOTE) consumed = true; st = P_VAL; break;
            case P_VAL: /* parseArgValue, state.go:95-153 */
                if constexpr (TYPED) { /* SetArgument (marker.go:53-63, argument.go:91-127) on the value strconv produced */
                    const uint32_t vk = k == OBM_K_SYNTHETIC_BOOL || k == OBM_K_BOOL_LITERAL ? 0u : k == OBM_K_INTEGER_LITERAL ? 1u
                                      : k == OBM_K_FLOAT_LITERAL ? 2u : k == OBM_K_STRING_LITERAL ? 3u : 4u;
                    const bool strconv_err = k == OBM_K_BOOL_LITERAL ? !parse_bool_ok(doc + off, len) : k == OBM_K_FLOAT_LITERAL && float32_overflows(doc + off, len);
                    const uint32_t out = vk < 4 && !strconv_err ? setarg_outcome(R.type[S.a_idx], vk, doc + off, len) : 0u;
                    if (out) { /* p.error: parser.current is the literal, or for the peeked synthetic bool the lexeme before it */
                        const bool syn = k == OBM_K_SYNTHETIC_BOOL;
                        if (!syn && len) { if (sc_any && !sc_nl && off == sc_off + sc_len) sc_len += len; else sc_broken = true; }
                        if (sc_broken) { S.nres = 0; S.nargs = 0; S.result(doc_id, i, 0, 0, 0xFFFFu, 0, 0, OBM_R_HOST, 0); return; }
                        S.nargs -= n_args;
                        const uint64_t ab = S.arg_at + S.nargs;
                        S.arg(syn ? cur_line : line, S.a_idx - R.arg_first[def], vk, off, syn ? 0u : len, syn ? (uint32_t)OBM_A_SYNTHETIC_TRUE : 0u);
                        S.result(doc_id, syn ? cur_tuple : i, sc_off, sc_len, (uint32_t)def, 1, ab, out == 2 ? OBM_R_PANIC : OBM_R_ERR_SETARG,
                                 syn ? cur_col : off - base + 1);
                        return;
                    }
                    if (vk < 4 && !strconv_err && R.typed[def]) { /* Fields[argName] = arg (marker.go:59): the last writer wins */
                        const uint32_t j = S.a_idx - R.arg_first[def];
                        const uint32_t sh = 16u * (j & 3u);
                        const uint32_t prev = j < 4 ? (uint32_t)(S.last >> sh) & 0xFFFFu : S.last4;
                        if ((S.set_mask >> j) & 1u) S.supersede((uint32_t)(arg_base - S.arg_at) + prev);
                        if (j < 4) S.last = (S.last & ~(0xFFFFull << sh)) | ((uint64_t)(n_args & 0xFFFFu) << sh); else S.last4 = n_args;
                        S.set_mask |= 1u << j;
                    }
                }
                if (k == OBM_K_SYNTHETIC_BOOL) { consumed = true; append = false; S.arg(a_off, a_len, 0, off, 0, OBM_A_SYNTHETIC_TRUE); n_args++; st = P_MORE; }
                else if (k == OBM_K_BOOL_LITERAL || k == OBM_K_FLOAT_LITERAL) {
                    consumed = true;
                    const bool bad = k == OBM_K_BOOL_LITERAL ? !parse_bool_ok(doc + off, len) : float32_overflows(doc + off, len);
                    if (bad) { /* error.go:8-22: the error Result carries scopeBuffer INCLUDING this lexeme and parser.current = it */
                        if (sc_any && !sc_nl && off == sc_off + sc_len) sc_len += len; else sc_broken = true;
                        if (sc_broken) { S.nres = 0; S.nargs = 0; S.result(doc_id, i, 0, 0, 0xFFFFu, 0, 0, OBM_R_HOST, 0); return; }
                        S.nargs -= n_args;
                        const uint64_t ab = S.arg_at + S.nargs;
                        S.arg(line, 0, k == OBM_K_BOOL_LITERAL ? 0u : 2u, off, len, 0);
                        S.result(doc_id, i, sc_off, sc_len, (uint32_t)def, 1, ab, k == OBM_K_BOOL_LITERAL ? OBM_R_ERR_PARSEBOOL : OBM_R_ERR_FLOAT32, off - base + 1);
                        return;
                    }
                    S.arg(a_off, a_len, k == OBM_K_BOOL_LITERAL ? 0u : 2u, off, len, 0); n_args++; st = P_MORE;
                } else if (k == OBM_K_INTEGER_LITERAL) { consumed = true; S.arg(a_off, a_len, 1, off, len, 0); n_args++; st = P_MORE; }
                else if (k == OBM_K_STRING_LITERAL) { consumed = true; S.arg(a_off, a_len, 3, off, len, 0); n_args++; st = P_VQ; }
                else st = P_PARSE;
                break;
            case P_VQ: if (k == OBM_K_QUOTE) consumed = true; st = P_MORE; break;
            default: /* P_MORE, state.go:155-169 */
                if (k == OBM_K_ARG_DELIMITER) { consumed = true; st = P_ARG; }
                else if (k == OBM_K_MARKER_END) { consumed = true; st = P_PARSE; }
                else st = P_PARSE;
                break;
            }
            /* arguments collected for a marker that is abandoned (unknown argument, unexpected lexeme) are dropped */
            if (st == P_PARSE && was != P_PARSE && def >= 0 && !(was == P_MORE && k == OBM_K_MARKER_END && consumed)) { S.nargs -= n_args; n_args = 0; def = -1; }
            if (consumed) {
                /* next(): the lexeme becomes parser.current and its Value is appended to scopeBuffer (position.go:7-20) */
                const bool synthetic = (k == OBM_K_SYNTHETIC_BOOL || k == OBM_K_MARKER_END || k == OBM_K_EOF);
                if (append) {
                    cur_tuple = i; cur_line = synthetic ? 0u : line; cur_col = synthetic ? 0u : off - base + 1u;
                    if (k == OBM_K_MARKER_END) { if (sc_nl) sc_broken = true; sc_nl = true; if (!sc_any) { sc_any = true; sc_off = off; sc_len = 0; } }
                    else if (k == OBM_K_SYNTHETIC_BOOL) sc_broken = true;
                    else if (len) {
                        if (!sc_any) { sc_any = true; sc_off = off; sc_len = len; }
                        else if (sc_nl || off != sc_off + sc_len) sc_broken = true;
                        else sc_len += len;
                    }
                }
                if (was == P_PARSE && st == P_PARSE && k != OBM_K_COMMENT) { sc_any = false; sc_nl = false; sc_len = 0; sc_broken = false; } /* the catch-all of parse */
                if (was == P_MORE && k == OBM_K_MARKER_END) { /* emit.go:8-24 */
                    if (sc_broken) { S.nres = 0; S.nargs = 0; S.result(doc_id, i, 0, 0, 0xFFFFu, 0, 0, OBM_R_HOST, 0); return; }
                    if constexpr (TYPED) { /* InflateObject (marker.go:65-95): parser.current is the synthetic MarkerEnd, {line:0 column:0} */
                        const uint32_t miss = R.required[def] & ~S.set_mask;
                        if (miss) { S.nargs -= n_args; S.result(doc_id, i, sc_off, sc_len, (uint32_t)def, 0, S.arg_at + S.nargs, OBM_R_ERR_MISSING | OBM_R_NL, miss); return; }
                    }
                    S.result(doc_id, marker_tuple, sc_off, sc_len, (uint32_t)def, n_args, arg_base, OBM_R_OK | OBM_R_NL, 0);
                    sc_any = false; sc_nl = false; sc_len = 0; sc_broken = false; def = -1; n_args = 0;
                }
            }
        }
        if (stop) break;
    }
    (void)cur_tuple; (void)cur_line; (void)cur_col;
}

} /* namespace obmr */
#endif
