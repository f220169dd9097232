/*
 * obm_decode.cpp -- host-side consumer of the tuple stream: replays one document's tuples as the
 * exact Lexeme{Type, Value, Pos} sequence of the reference lexer.  No lexing happens here; the
 * tuples come from the GPU (obm_lex_batch).
 *
 * Mirrors the consumer-facing surface of internal/markers/lexer (lexer.go:27-53, lexeme.go:32-36):
 *   obm_stream_new  ~ NewLexer + Run      obm_stream_next ~ NextLexeme (zero Lexeme once closed)
 * and reproduces the reference's message formats:
 *   error.go:18,40   "%s at position: %+v, following %q"
 *   state.go:193     "unmatched string delimiter %s at position %+v, following %q"
 *   state.go:259,270 "invalid float|integer literal %q: %s before position %d"
 * `%q` is strconv.Quote (obm_quote.h), `%+v`/`%d` of position{line,column} print {line:L column:C} / {L C}.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>

#include "../../include/obmarkers.h"
#include "go_unicode_tables.h"
#include "obm_core.h"
#include "obm_quote.h"

namespace {

const char F64_OVERFLOW_DIGITS[] = GO_F64_OVERFLOW_DIGITS;

const obm::Tables &host_tables() {
    static const obm::Tables T = { GO_LETTER_RANGES, GO_LETTER_RANGES_N, GO_NUMBER_RANGES, GO_NUMBER_RANGES_N, F64_OVERFLOW_DIGITS };
    return T;
}

/* Each invalid byte of input becomes U+FFFD in a Value: next() does `buffer += string(r)` with
 * r == utf8.RuneError (position.go:21,36). */
void append_sanitized(std::string &dst, const uint8_t *p, uint64_t n) {
    uint64_t i = 0, run = 0;
    while (i < n) {
        if (p[i] < 0x80) { i++; continue; }
        uint32_t w; int r = obm::decode_rune(p, (uint32_t)i, (uint32_t)(n > 0xFFFFFFFFull ? 0xFFFFFFFFu : n), w);
        if (r == obm::RUNE_ERR && w == 1) {
            dst.append((const char *)p + run, i - run);
            dst.append("\xEF\xBF\xBD");
            i += 1; run = i;
        } else i += w;
    }
    dst.append((const char *)p + run, n - run);
}

struct Basis { uint64_t line; uint64_t base; uint64_t drift; };

} // namespace

struct obm_stream {
    const uint8_t *doc; uint64_t n;
    const obm_tuple *t; uint64_t nt, i;
    std::string pending;             /* the reference lexer's un-emitted `buffer` */
    uint64_t chain_start, chain_end; /* contiguous PART chain: where `start` really is */
    Basis chain_basis;
    Basis basis;
    uint64_t linehi;
    std::string last_value;          /* lastEmittedLexeme.Value */
    int64_t last_line, last_col;     /* lastEmittedLexeme.Pos */
    std::string cur;                 /* storage for the lexeme being returned */
    bool closed;
};

static int64_t col_of(const Basis &b, uint64_t off) { return (int64_t)off - (int64_t)b.base + 1 - (int64_t)b.drift; }

extern "C" obm_stream *obm_stream_new(const uint8_t *doc, uint64_t doc_len, const obm_tuple *tuples, uint64_t ntuples) {
    obm_stream *s = new (std::nothrow) obm_stream();
    if (!s) return nullptr;
    s->doc = doc; s->n = doc_len; s->t = tuples; s->nt = ntuples; s->i = 0;
    s->chain_start = s->chain_end = 0; s->chain_basis = Basis{1, 0, 0};
    s->basis = Basis{1, 0, 0}; s->linehi = 0;
    s->last_line = s->last_col = 0; s->closed = false;
    return s;
}

extern "C" void obm_stream_free(obm_stream *s) { delete s; }

static void put_pos(std::string &o, bool plus_v, int64_t line, int64_t col) {
    char tmp[96];
    if (plus_v) snprintf(tmp, sizeof tmp, "{line:%lld column:%lld}", (long long)line, (long long)col);
    else snprintf(tmp, sizeof tmp, "{%lld %lld}", (long long)line, (long long)col);
    o += tmp;
}

extern "C" int obm_stream_next(obm_stream *s, obm_lexeme *out) {
    out->type = 0; out->value = (const uint8_t *)""; out->value_len = 0; out->line = 0; out->column = 0;
    if (s->closed) return 0;
    while (s->i < s->nt) {
        obm_tuple tu = s->t[s->i++];
        unsigned kind = OBM_TUPLE_KIND(tu);
        uint64_t off = OBM_TUPLE_OFF(tu), len = OBM_TUPLE_LEN(tu);
        const bool slices = kind == OBM_K_PART || kind == OBM_K_ERR_FLOAT || kind == OBM_K_ERR_INT ||
                            (kind >= OBM_K_COMMENT && kind <= OBM_K_QUOTE);
        if (slices) { /* never read outside the document, whatever the tuple says */
            if (off > s->n) off = s->n;
            if (off + len > s->n) len = s->n - off;
        }
        switch (kind) {
        case OBM_K_LINEHI: s->linehi = off; continue;
        case OBM_K_LINE: s->basis = Basis{(s->linehi << OBM_LEN_BITS) | len, off, 0}; s->linehi = 0; continue;
        case OBM_K_DRIFT: s->basis.drift += 1; continue;
        case OBM_K_FLUSH: s->pending.clear(); continue;
        case OBM_K_PART:
            if (s->pending.empty() || s->chain_end != off) { s->chain_start = off; s->chain_basis = s->basis; }
            append_sanitized(s->pending, s->doc + off, len);
            s->chain_end = off + len;
            continue;
        case OBM_K_SYNTHETIC_BOOL: case OBM_K_MARKER_END: case OBM_K_EOF: {
            s->cur = kind == OBM_K_SYNTHETIC_BOOL ? "true" : kind == OBM_K_MARKER_END ? "\n" : "";
            s->last_value = s->cur; s->last_line = 0; s->last_col = 0;
            out->type = (int32_t)kind; out->value = (const uint8_t *)s->cur.data(); out->value_len = s->cur.size();
            if (kind == OBM_K_EOF) s->closed = true;
            return 1;
        }
        case OBM_K_WARN_NOSCOPE: case OBM_K_WARN_INVALID: case OBM_K_ERR_MALFORMED: {
            int64_t line = (int64_t)s->basis.line, col = col_of(s->basis, off);
            std::string v = kind == OBM_K_WARN_NOSCOPE ? "marker without scope found"
                          : kind == OBM_K_WARN_INVALID ? "invalid marker found" : "malformed argument: " + s->pending;
            v += " at position: "; put_pos(v, true, line, col);
            v += ", following "; obm::go_quote(v, s->last_value + s->pending);
            s->cur.swap(v);
            out->type = kind == OBM_K_ERR_MALFORMED ? OBM_K_ERROR : OBM_K_WARNING;
            out->value = (const uint8_t *)s->cur.data(); out->value_len = s->cur.size(); out->line = line; out->column = col;
            if (kind == OBM_K_ERR_MALFORMED) s->closed = true;
            return 1;
        }
        case OBM_K_ERR_UNMATCHED: {
            /* pos/context were captured right after the opening quote (state.go:193-194) */
            std::string v = "unmatched string delimiter ";
            v += s->last_value.empty() ? std::string("?") : s->last_value.substr(s->last_value.size() - 1);
            v += " at position "; put_pos(v, true, s->last_line, s->last_col + 1);
            v += ", following "; obm::go_quote(v, s->last_value);
            s->cur.swap(v);
            out->type = OBM_K_ERROR; out->value = (const uint8_t *)s->cur.data(); out->value_len = s->cur.size();
            out->line = (int64_t)s->basis.line; out->column = col_of(s->basis, off);
            s->closed = true;
            return 1;
        }
        case OBM_K_ERR_FLOAT: case OBM_K_ERR_INT: {
            std::string lit = s->pending; append_sanitized(lit, s->doc + off, len);
            const bool isf = kind == OBM_K_ERR_FLOAT;
            int code = isf ? obm::parse_float_err(host_tables(), (const uint8_t *)lit.data(), (uint32_t)lit.size())
                           : obm::atoi_err((const uint8_t *)lit.data(), (uint32_t)lit.size());
            int64_t line = (int64_t)s->basis.line, col = col_of(s->basis, off + len);
            std::string v = isf ? "invalid float literal " : "invalid integer literal ";
            obm::go_quote(v, lit);
            v += isf ? ": strconv.ParseFloat: parsing " : ": strconv.Atoi: parsing ";
            obm::go_quote(v, lit);
            v += code == 2 ? ": value out of range" : ": invalid syntax";
            v += " before position "; put_pos(v, false, line, col);
            s->cur.swap(v);
            out->type = OBM_K_ERROR; out->value = (const uint8_t *)s->cur.data(); out->value_len = s->cur.size();
            out->line = line; out->column = col;
            s->closed = true;
            return 1;
        }
        default:
            if (kind >= OBM_K_COMMENT && kind <= OBM_K_QUOTE) {
                /* a real lexeme: Value = pending buffer + its own slice; Pos = `start` */
                bool chained = !s->pending.empty() && s->chain_end == off;
                const Basis &b = chained ? s->chain_basis : s->basis;
                uint64_t posoff = chained ? s->chain_start : off;
                s->cur.swap(s->pending); s->pending.clear();
                append_sanitized(s->cur, s->doc + off, len);
                s->last_value = s->cur; s->last_line = (int64_t)b.line; s->last_col = col_of(b, posoff);
                out->type = (int32_t)kind; out->value = (const uint8_t *)s->cur.data(); out->value_len = s->cur.size();
                out->line = s->last_line; out->column = s->last_col;
                return 1;
            }
            continue; /* kinds 0, 14..17, 19 never appear in a valid stream */
        }
    }
    s->closed = true;
    return 0;
}

extern "C" int64_t obm_decode_doc(const uint8_t *doc, uint64_t doc_len, const obm_tuple *tuples, uint64_t ntuples,
                                  uint8_t **out, uint64_t *out_len) {
    obm_stream *s = obm_stream_new(doc, doc_len, tuples, ntuples);
    if (!s) return OBM_E_NOMEM;
    std::string buf;
    int64_t count = 0;
    obm_lexeme lx;
    while (obm_stream_next(s, &lx)) {
        uint8_t hdr[13];
        uint32_t ln = (uint32_t)lx.line, co = (uint32_t)lx.column, vl = (uint32_t)lx.value_len;
        hdr[0] = (uint8_t)lx.type; memcpy(hdr + 1, &ln, 4); memcpy(hdr + 5, &co, 4); memcpy(hdr + 9, &vl, 4);
        buf.append((const char *)hdr, 13);
        buf.append((const char *)lx.value, lx.value_len);
        count++;
    }
    obm_stream_free(s);
    uint8_t *p = (uint8_t *)malloc(buf.size() ? buf.size() : 1);
    if (!p) return OBM_E_NOMEM;
    memcpy(p, buf.data(), buf.size());
    *out = p; *out_len = buf.size();
    return count;
}

extern "C" void obm_free(void *p) { free(p); }
