/*
 * lexer_oracle.c -- CPU ORACLE (test infrastructure, NOT product code).
 *
 * A plain-C restatement of the reference marker lexer
 *   /root/reference/internal/markers/lexer/{lexer,lexeme,emit,error,stack,position,
 *                                           consume,discard,peek,state}.go
 * of vmware-tanzu-labs/operator-builder @ 2827f233, written function by function so that each
 * routine can be read against the Go source it follows (cited as file:line below).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this file's shared object.  The product (libobmarkers.so) never links or calls it.
 *
 * The arithmetic the reference relies on lives in the Go 1.16 standard library (go.mod:3), which
 * is not vendored under /root/reference and cannot be built here (no Go toolchain):
 *   bufio.Reader  (default 4096-byte buffer; Peek/Discard/ReadRune/UnreadRune)  -> bufreader_* below,
 *   unicode/utf8  (DecodeRune, RuneLen)                                          -> go_decode_rune, go_rune_len,
 *   unicode       (IsSpace/IsLetter/IsNumber, Unicode 13.0 tables)               -> go_unicode_tables.h (generated from
 *                                                                                  tests/golden/unicode13.json),
 *   strconv       (ParseFloat(.,64), Atoi, Quote)                                -> go_parse_float_err, go_atoi_err, go_quote,
 *   fmt           (%s %q %d %+v of the shapes used in error.go / state.go)       -> hand formatted.
 * Those are restated from their published behaviour.
 *
 * PARITY PINNING: this oracle is pinned against the reference's own 24 golden vectors
 * (lexer/lexer_test.go:28-402) and its primitive tests (consume_internal_test.go,
 * peek_internal_test.go) -- see tests/test_oracle_golden.py.  Lexeme positions, error texts,
 * float/bool literals, multi-marker lines and non-ASCII input are NOT covered by any reference
 * test; for those this file is "parity unpinned" (derived from source reading only).
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>

#include "go_unicode_tables.h"

/* ------------------------------------------------------------------------------------------ */
/* growable byte string (Go `string` / `[]byte` stand-in)                                      */
/* ------------------------------------------------------------------------------------------ */
typedef struct { uint8_t *p; size_t len, cap; } gstr;

static void gs_reserve(gstr *s, size_t extra) {
    if (s->len + extra <= s->cap) return;
    size_t nc = s->cap ? s->cap * 2 : 64;
    while (nc < s->len + extra) nc *= 2;
    s->p = (uint8_t *)realloc(s->p, nc);
    s->cap = nc;
}
static void gs_append(gstr *s, const void *b, size_t n) { gs_reserve(s, n); memcpy(s->p + s->len, b, n); s->len += n; }
static void gs_appendc(gstr *s, uint8_t c) { gs_reserve(s, 1); s->p[s->len++] = c; }
static void gs_appends(gstr *s, const char *z) { gs_append(s, z, strlen(z)); }
static void gs_clear(gstr *s) { s->len = 0; }
static void gs_free(gstr *s) { free(s->p); s->p = NULL; s->len = s->cap = 0; }

/* ------------------------------------------------------------------------------------------ */
/* unicode/utf8                                                                                */
/* ------------------------------------------------------------------------------------------ */
#define RUNE_ERROR 0xFFFD
#define RUNE_EOF (-1) /* lexeme.go:38 */

/* utf8.DecodeRune: (RuneError,0) on empty, (RuneError,1) on any invalid or short encoding. */
static int32_t go_decode_rune(const uint8_t *b, size_t n, int *width) {
    if (n == 0) { *width = 0; return RUNE_ERROR; }
    uint8_t c0 = b[0];
    if (c0 < 0x80) { *width = 1; return c0; }
    if (c0 < 0xC2 || c0 > 0xF4) { *width = 1; return RUNE_ERROR; }
    if (c0 < 0xE0) {
        if (n < 2 || (b[1] & 0xC0) != 0x80) { *width = 1; return RUNE_ERROR; }
        *width = 2; return ((int32_t)(c0 & 0x1F) << 6) | (b[1] & 0x3F);
    }
    if (c0 < 0xF0) {
        uint8_t lo = 0x80, hi = 0xBF;
        if (c0 == 0xE0) lo = 0xA0; else if (c0 == 0xED) hi = 0x9F;
        if (n < 3 || b[1] < lo || b[1] > hi || (b[2] & 0xC0) != 0x80) { *width = 1; return RUNE_ERROR; }
        *width = 3; return ((int32_t)(c0 & 0x0F) << 12) | ((int32_t)(b[1] & 0x3F) << 6) | (b[2] & 0x3F);
    }
    {
        uint8_t lo = 0x80, hi = 0xBF;
        if (c0 == 0xF0) lo = 0x90; else if (c0 == 0xF4) hi = 0x8F;
        if (n < 4 || b[1] < lo || b[1] > hi || (b[2] & 0xC0) != 0x80 || (b[3] & 0xC0) != 0x80) { *width = 1; return RUNE_ERROR; }
        *width = 4;
        return ((int32_t)(c0 & 0x07) << 18) | ((int32_t)(b[1] & 0x3F) << 12) | ((int32_t)(b[2] & 0x3F) << 6) | (b[3] & 0x3F);
    }
}

/* utf8.FullRune */
static int go_full_rune(const uint8_t *b, size_t n) {
    if (n == 0) return 0;
    uint8_t c0 = b[0];
    if (c0 < 0x80 || c0 < 0xC2 || c0 > 0xF4) return 1; /* ASCII or invalid lead: "full" (decodes as width 1) */
    size_t need = c0 < 0xE0 ? 2 : (c0 < 0xF0 ? 3 : 4);
    if (n >= need) return 1;
    /* short: full only if already known invalid */
    uint8_t lo = 0x80, hi = 0xBF;
    if (c0 == 0xE0) lo = 0xA0; else if (c0 == 0xED) hi = 0x9F; else if (c0 == 0xF0) lo = 0x90; else if (c0 == 0xF4) hi = 0x8F;
    if (n > 1 && (b[1] < lo || b[1] > hi)) return 1;
    if (n > 2 && (b[2] & 0xC0) != 0x80) return 1;
    return 0;
}

/* utf8.RuneLen */
static int go_rune_len(int32_t r) {
    if (r < 0) return -1;
    if (r < 0x80) return 1;
    if (r < 0x800) return 2;
    if (r >= 0xD800 && r <= 0xDFFF) return -1;
    if (r < 0x10000) return 3;
    if (r <= 0x10FFFF) return 4;
    return -1;
}

/* string(rune): invalid runes become U+FFFD */
static void gs_append_rune(gstr *s, int32_t r) {
    if (r < 0 || r > 0x10FFFF || (r >= 0xD800 && r <= 0xDFFF)) r = RUNE_ERROR;
    if (r < 0x80) gs_appendc(s, (uint8_t)r);
    else if (r < 0x800) { gs_appendc(s, 0xC0 | (r >> 6)); gs_appendc(s, 0x80 | (r & 0x3F)); }
    else if (r < 0x10000) { gs_appendc(s, 0xE0 | (r >> 12)); gs_appendc(s, 0x80 | ((r >> 6) & 0x3F)); gs_appendc(s, 0x80 | (r & 0x3F)); }
    else { gs_appendc(s, 0xF0 | (r >> 18)); gs_appendc(s, 0x80 | ((r >> 12) & 0x3F)); gs_appendc(s, 0x80 | ((r >> 6) & 0x3F)); gs_appendc(s, 0x80 | (r & 0x3F)); }
}

/* ------------------------------------------------------------------------------------------ */
/* unicode predicates                                                                          */
/* ------------------------------------------------------------------------------------------ */
static int in_ranges(const unsigned int (*t)[2], int n, int32_t r) {
    if (r < 0) return 0;
    int lo = 0, hi = n - 1;
    while (lo <= hi) {
        int mid = (lo + hi) >> 1;
        if ((unsigned)r < t[mid][0]) hi = mid - 1;
        else if ((unsigned)r > t[mid][1]) lo = mid + 1;
        else return 1;
    }
    return 0;
}
static int go_is_space(int32_t r) { return in_ranges(GO_SPACE_RANGES, GO_SPACE_RANGES_N, r); }
static int go_is_letter(int32_t r) { return in_ranges(GO_LETTER_RANGES, GO_LETTER_RANGES_N, r); }
static int go_is_number(int32_t r) { return in_ranges(GO_NUMBER_RANGES, GO_NUMBER_RANGES_N, r); }
static int go_is_print(int32_t r) { return in_ranges(GO_PRINT_RANGES, GO_PRINT_RANGES_N, r); }

/* ------------------------------------------------------------------------------------------ */
/* strconv.Quote (what fmt's %q applies to a string)                                           */
/* ------------------------------------------------------------------------------------------ */
static void go_quote(gstr *out, const uint8_t *s, size_t n) {
    static const char hex[] = "0123456789abcdef";
    gs_appendc(out, '"');
    size_t i = 0;
    while (i < n) {
        int w = 1;
        int32_t r = s[i];
        if (r >= 0x80) r = go_decode_rune(s + i, n - i, &w);
        if (w == 1 && r == RUNE_ERROR) {
            gs_appends(out, "\\x"); gs_appendc(out, hex[s[i] >> 4]); gs_appendc(out, hex[s[i] & 0xF]);
            i += 1; continue;
        }
        if (r == '"' || r == '\\') { gs_appendc(out, '\\'); gs_appendc(out, (uint8_t)r); i += w; continue; }
        if (go_is_print(r)) { gs_append(out, s + i, w); i += w; continue; }
        switch (r) {
        case '\a': gs_appends(out, "\\a"); break;
        case '\b': gs_appends(out, "\\b"); break;
        case '\f': gs_appends(out, "\\f"); break;
        case '\n': gs_appends(out, "\\n"); break;
        case '\r': gs_appends(out, "\\r"); break;
        case '\t': gs_appends(out, "\\t"); break;
        case '\v': gs_appends(out, "\\v"); break;
        default:
            if (r < ' ') { gs_appends(out, "\\x"); gs_appendc(out, hex[(r >> 4) & 0xF]); gs_appendc(out, hex[r & 0xF]); }
            else if (r < 0x10000) { gs_appends(out, "\\u"); for (int sft = 12; sft >= 0; sft -= 4) gs_appendc(out, hex[(r >> sft) & 0xF]); }
            else { gs_appends(out, "\\U"); for (int sft = 28; sft >= 0; sft -= 4) gs_appendc(out, hex[(r >> sft) & 0xF]); }
        }
        i += w;
    }
    gs_appendc(out, '"');
}

/* ------------------------------------------------------------------------------------------ */
/* strconv.ParseFloat(s, 64) / strconv.Atoi(s): only the error outcome matters to the lexer    */
/* (state.go:258, 269).  Returns 0 = ok, 1 = "invalid syntax", 2 = "value out of range".      */
/* ------------------------------------------------------------------------------------------ */
static int lower(int c) { return c | 0x20; }

/* 2^1024 - 2^970: the smallest decimal that rounds (half-even) to +Inf in float64. */
static const char FLOAT64_OVERFLOW_DIGITS[] =
    "1797693134862315807937289714053034150799341327100378269361737789804449682927647509466490179775872070963"
    "3028641669288791094655554785194040263065748867150582068190890200070838367627385484581771153176447573027"
    "0069855571366959622842914819860834936475292719074168444365510704342711559699508093042880177904174497792";

static int go_parse_float_err(const uint8_t *s, size_t n) {
    size_t i = 0;
    if (n == 0) return 1;
    /* special(): [+-]?(inf|infinity) or nan, case-insensitive (atof.go special) */
    {
        size_t j = 0; int c0 = s[0];
        if (c0 == '+' || c0 == '-') j = 1;
        if (j < n && (j == 1 || lower(c0) == 'i') ) {
            const char *inf = "infinity"; size_t k = 0;
            while (j + k < n && k < 8 && lower(s[j + k]) == inf[k]) k++;
            if (k > 3 && k < 8) k = 3;
            if (k == 3 || k == 8) return (j + k == n) ? 0 : 1;
        } else if (lower(c0) == 'n') {
            if (n >= 3 && lower(s[1]) == 'a' && lower(s[2]) == 'n') return n == 3 ? 0 : 1;
        }
    }
    int underscores = 0;
    if (s[i] == '+' || s[i] == '-') i++;
    int base = 10; int expChar = 'e';
    if (i + 2 < n && s[i] == '0' && lower(s[i + 1]) == 'x') { base = 16; i += 2; expChar = 'p'; }
    int sawdot = 0, sawdigits = 0;
    long long nd = 0, dp = 0;
    size_t digits_begin = i;
    int mant_nonzero = 0;
    for (; i < n; i++) {
        int c = s[i];
        if (c == '_') { underscores = 1; continue; }
        if (c == '.') { if (sawdot) break; sawdot = 1; dp = nd; continue; }
        if (c >= '0' && c <= '9') {
            sawdigits = 1;
            if (c == '0' && nd == 0) { dp--; continue; }
            nd++; mant_nonzero = 1; continue;
        }
        if (base == 16 && lower(c) >= 'a' && lower(c) <= 'f') { sawdigits = 1; nd++; mant_nonzero = 1; continue; }
        break;
    }
    size_t digits_end = i;
    if (!sawdigits) return 1;
    if (!sawdot) dp = nd;
    if (base == 16) dp *= 4;
    if (i < n && lower(s[i]) == expChar) {
        i++;
        if (i >= n) return 1;
        int esign = 1;
        if (s[i] == '+') i++; else if (s[i] == '-') { i++; esign = -1; }
        if (i >= n || s[i] < '0' || s[i] > '9') return 1;
        long long e = 0;
        for (; i < n && ((s[i] >= '0' && s[i] <= '9') || s[i] == '_'); i++) {
            if (s[i] == '_') { underscores = 1; continue; }
            if (e < 10000) e = e * 10 + (s[i] - '0');
        }
        dp += e * esign;
    } else if (base == 16) return 1;
    if (underscores) return 1; /* underscoreOK needs a base prefix AND base==0 semantics; never ok for "0x_"-less input; the
                                  lexer's numeric alphabet has no '_' or 'x' anyway */
    if (i != n) return 1;
    if (base == 16) return 0; /* unreachable from the lexer (no 'x' in its numeric alphabet) */
    if (!mant_nonzero) return 0;
    /* value = 0.d1d2d3... * 10^dp with d1 != 0 (leading zeros were skipped above) */
    if (dp > 309) return 2;
    if (dp < 309) return 0;
    /* dp == 309: compare significant digits with 2^1024-2^970 (309 digits); >= means overflow */
    {
        size_t k = 0; int started = 0;
        for (size_t j = digits_begin; j < digits_end; j++) {
            int c = s[j];
            if (c == '.' || c == '_') continue;
            if (!started) { if (c == '0') continue; started = 1; }
            if (k < 309) {
                int t = FLOAT64_OVERFLOW_DIGITS[k];
                if (c > t) return 2;
                if (c < t) return 0;
                k++;
            } else {
                return 2; /* equal on 309 digits, more digits follow: >= threshold either way */
            }
        }
        /* ran out of input digits: remaining input digits are implicit zeros */
        for (; k < 309; k++) if (FLOAT64_OVERFLOW_DIGITS[k] != '0') return 0;
        return 2;
    }
}

static int go_atoi_err(const uint8_t *s, size_t n) {
    /* strconv.Atoi == ParseInt(s, 10, 0) with int = int64 (the <19-byte fast path gives the same
     * outcomes).  ParseUint reports overflow the moment it happens, i.e. BEFORE a later bad byte. */
    size_t i = 0; int neg = 0;
    if (n == 0) return 1;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
    if (i >= n) return 1;
    const uint64_t cutoff = 0xFFFFFFFFFFFFFFFFULL / 10 + 1;
    uint64_t v = 0;
    for (; i < n; i++) {
        if (s[i] < '0' || s[i] > '9') return 1; /* includes '_' (legal only with base 0) and non-ASCII */
        if (v >= cutoff) return 2;
        v *= 10;
        uint64_t v1 = v + (uint64_t)(s[i] - '0');
        if (v1 < v) return 2;
        v = v1;
    }
    if (!neg && v >= (1ULL << 63)) return 2;
    if (neg && v > (1ULL << 63)) return 2;
    return 0;
}

/* ------------------------------------------------------------------------------------------ */
/* bufio.Reader (Go 1.16 src/bufio/bufio.go) over a bytes.Buffer                               */
/* ------------------------------------------------------------------------------------------ */
#define BUFIO_SIZE 4096
typedef struct {
    const uint8_t *src; size_t srclen, srcpos; /* the underlying bytes.Buffer */
    uint8_t buf[BUFIO_SIZE];
    int r, w;
    int err;          /* 0 = nil, 1 = io.EOF (sticky until readErr()) */
    int lastRuneSize; /* -1 = invalid */
} bufreader;

static void br_init(bufreader *b, const uint8_t *src, size_t n) {
    b->src = src; b->srclen = n; b->srcpos = 0; b->r = b->w = 0; b->err = 0; b->lastRuneSize = -1;
}
/* bytes.Buffer.Read: (0, io.EOF) when empty, else copies min(len(p), remaining) */
static void br_fill(bufreader *b) {
    if (b->r > 0) { memmove(b->buf, b->buf + b->r, (size_t)(b->w - b->r)); b->w -= b->r; b->r = 0; }
    for (int i = 100; i > 0; i--) {
        size_t room = (size_t)(BUFIO_SIZE - b->w);
        size_t rem = b->srclen - b->srcpos;
        if (rem == 0) { b->err = 1; return; }
        size_t n = rem < room ? rem : room;
        memcpy(b->buf + b->w, b->src + b->srcpos, n);
        b->srcpos += n; b->w += (int)n;
        if (n > 0) return;
    }
}
/* Peek(n): returns pointer/len into buf; invalidates UnreadRune */
static const uint8_t *br_peek(bufreader *b, long long n, int *outlen) {
    b->lastRuneSize = -1;
    while (b->w - b->r < n && b->w - b->r < BUFIO_SIZE && b->err == 0) br_fill(b);
    if (n > BUFIO_SIZE) { *outlen = b->w - b->r; return b->buf + b->r; }
    int avail = b->w - b->r;
    if (avail < n) { n = avail; b->err = 0; /* readErr() clears it */ }
    *outlen = (int)n;
    return b->buf + b->r;
}
/* Discard(n) -- Go 1.16 does NOT invalidate UnreadRune here (added in 1.18); irrelevant to the
 * lexer because every Discard is preceded by a Peek (discard.go:18,28). */
static int br_discard(bufreader *b, int n) {
    if (n <= 0) return 0;
    int remain = n;
    for (;;) {
        int skip = b->w - b->r;
        if (skip == 0) { br_fill(b); skip = b->w - b->r; }
        if (skip > remain) skip = remain;
        b->r += skip; remain -= skip;
        if (remain == 0) return n;
        if (b->err != 0) { b->err = 0; return n - remain; }
    }
}
/* ReadRune: returns rune and size; size 0 + *eof=1 at end of input */
static int32_t br_read_rune(bufreader *b, int *size, int *eof) {
    while (b->r + 4 > b->w && !go_full_rune(b->buf + b->r, (size_t)(b->w - b->r)) && b->err == 0 && b->w - b->r < BUFIO_SIZE) br_fill(b);
    b->lastRuneSize = -1;
    if (b->r == b->w) { b->err = 0; *size = 0; *eof = 1; return 0; }
    *eof = 0;
    int32_t r = b->buf[b->r]; int sz = 1;
    if (r >= 0x80) r = go_decode_rune(b->buf + b->r, (size_t)(b->w - b->r), &sz);
    b->r += sz; b->lastRuneSize = sz; *size = sz;
    return r;
}
static void br_unread_rune(bufreader *b) {
    if (b->lastRuneSize < 0 || b->r < b->lastRuneSize) return; /* ErrInvalidUnreadRune, ignored at position.go:56 */
    b->r -= b->lastRuneSize; b->lastRuneSize = -1;
}

/* ------------------------------------------------------------------------------------------ */
/* Lexeme / Lexer (lexeme.go:6-36, lexer.go:12-24)                                             */
/* ------------------------------------------------------------------------------------------ */
enum {
    LexemeError = 0, LexemeComment, LexemeMarkerStart, LexemeScope, LexemeSeparator, LexemeArg,
    LexemeArgAssignment, LexemeArgDelimiter, LexemeStringLiteral, LexemeFloatLiteral,
    LexemeIntegerLiteral, LexemeSyntheticBoolLiteral, LexemeBoolLiteral, LexemeQuote,
    LexemeSliceBegin, LexemeSliceEnd, LexemeSliceDelimiter, LexemeNakedSliceDelimiter,
    LexemeMarkerEnd, LexemeWarning, LexemeEOF
};

typedef struct { long long line, column; } position;

/* sink: what `l.items <- lx` delivers to */
typedef struct {
    int mode;            /* 0 = serialise every lexeme, 1 = count + hash only */
    gstr out;            /* mode 0: [u8 type][u32 line][u32 col][u32 vlen][value] ... */
    uint64_t n_lexemes, n_markers, hash;
} sink;

typedef enum {
    ST_NIL = 0, ST_lex, ST_lexCommentStart, ST_lexComment, ST_lexMarkerStart, ST_lexMarker,
    ST_lexArgs, ST_lexArgValueInitial, ST_lexFloatLiteral, ST_lexIntegerLiteral, ST_lexMoreArgs
} state_id;

typedef struct {
    gstr buffer;
    position start, pos;
    long long *lineLens; size_t lineLensCap; /* map[int]int, keyed by line number */
    int width;
    state_id stack[8]; int nstack;
    int lastType; gstr lastValue; /* lastEmittedLexeme (zero value: Type 0, Value "") */
    bufreader reader;
    sink *items;
} Lexer;

static uint64_t fnv1a(uint64_t h, const void *p, size_t n) {
    const uint8_t *b = (const uint8_t *)p;
    for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 0x100000001b3ULL; }
    return h;
}

static void send(Lexer *l, int typ, const uint8_t *v, size_t vlen, position pos) {
    sink *s = l->items;
    s->n_lexemes++;
    if (typ == LexemeMarkerStart) s->n_markers++;
    uint8_t hdr[13];
    uint32_t ln = (uint32_t)pos.line, co = (uint32_t)pos.column, vl = (uint32_t)vlen;
    hdr[0] = (uint8_t)typ; memcpy(hdr + 1, &ln, 4); memcpy(hdr + 5, &co, 4); memcpy(hdr + 9, &vl, 4);
    if (s->mode == 0) { gs_append(&s->out, hdr, 13); gs_append(&s->out, v, vlen); }
    else { s->hash = fnv1a(fnv1a(s->hash, hdr, 13), v, vlen); }
}

static void lineLens_set(Lexer *l, long long line, long long v) {
    if (line < 0) return;
    if ((size_t)line >= l->lineLensCap) {
        size_t nc = l->lineLensCap ? l->lineLensCap * 2 : 64;
        while (nc <= (size_t)line) nc *= 2;
        l->lineLens = (long long *)realloc(l->lineLens, nc * sizeof(long long));
        memset(l->lineLens + l->lineLensCap, 0, (nc - l->lineLensCap) * sizeof(long long));
        l->lineLensCap = nc;
    }
    l->lineLens[line] = v;
}
static long long lineLens_get(Lexer *l, long long line) {
    if (line < 0 || (size_t)line >= l->lineLensCap) return 0; /* missing map key -> zero value */
    return l->lineLens[line];
}

/* lexer.go:27-40 NewLexer */
static void lexer_init(Lexer *l, const uint8_t *doc, size_t n, sink *s) {
    memset(l, 0, sizeof *l);
    l->start.line = 1; l->start.column = 1;
    l->pos.line = 1; l->pos.column = 1;
    l->lastType = 0;
    l->items = s;
    br_init(&l->reader, doc, n);
}
static void lexer_free(Lexer *l) { gs_free(&l->buffer); gs_free(&l->lastValue); free(l->lineLens); }

/* position.go:60-65 resetPosition */
static void resetPosition(Lexer *l) {
    lineLens_set(l, l->pos.line, l->pos.column);
    l->pos.line++;
    l->pos.column = 1;
}

/* position.go:18-39 next */
static int32_t lx_next(Lexer *l) {
    int eof = 0;
    int32_t r = br_read_rune(&l->reader, &l->width, &eof);
    if (eof) { l->width = 0; return RUNE_EOF; }
    if (r == '\n') resetPosition(l); else l->pos.column += l->width;
    gs_append_rune(&l->buffer, r);
    return r;
}

/* position.go:43-57 backup */
static void lx_backup(Lexer *l) {
    if (l->width != 0) {
        l->pos.column -= l->width;
        if (l->buffer.len != 0) l->buffer.len -= 1;
    }
    if (l->pos.column == 0 && l->pos.line > 1) {
        l->pos.line--;
        l->pos.column = lineLens_get(l, l->pos.line);
    }
    br_unread_rune(&l->reader);
}

/* peek.go:20-44 peekN; returns count written to rs (<= n), last may be RUNE_EOF */
static int lx_peekN(Lexer *l, long long n, int32_t **rs_out) {
    static __thread int32_t *rs = NULL; static __thread size_t rscap = 0;
    if ((size_t)n + 1 > rscap) { rscap = (size_t)n + 64; rs = (int32_t *)realloc(rs, rscap * sizeof(int32_t)); }
    int cnt = 0;
    l->width = 0;
    int blen = 0;
    const uint8_t *b = br_peek(&l->reader, n * 4, &blen);
    while (n > cnt) {
        if (blen == 0) { rs[cnt++] = RUNE_EOF; break; }
        int w; int32_t r = go_decode_rune(b, (size_t)blen, &w);
        b += w; blen -= w;
        l->width += w;
        rs[cnt++] = r;
    }
    *rs_out = rs;
    return cnt;
}
/* peek.go:14-16 peek */
static int32_t lx_peek(Lexer *l) { int32_t *rs; lx_peekN(l, 1, &rs); return rs[0]; }

/* strings.HasPrefix(string(runes), p): string([]rune) maps invalid runes (incl. -1) to U+FFFD */
static int runes_have_prefix(const int32_t *rs, int cnt, const char *p) {
    /* only the first strlen(p) bytes of string(runes) matter; each rune contributes >= 1 byte */
    size_t pl = strlen(p);
    uint8_t stackbuf[64]; gstr tmp = {0};
    int use = cnt < (int)pl ? cnt : (int)pl; /* runes needed to cover pl bytes */
    if ((size_t)use * 4 <= sizeof stackbuf) { tmp.p = stackbuf; tmp.cap = sizeof stackbuf; }
    for (int i = 0; i < use; i++) gs_append_rune(&tmp, rs[i]);
    int ok = tmp.len >= pl && memcmp(tmp.p, p, pl) == 0;
    if (tmp.p != stackbuf) gs_free(&tmp);
    return ok;
}
/* peek.go:92-96 hasPrefix -- len(p) is a BYTE length used as a rune count */
static int lx_hasPrefix(Lexer *l, const char *p) {
    int32_t *rs; int cnt = lx_peekN(l, (long long)strlen(p), &rs);
    return runes_have_prefix(rs, cnt, p);
}
/* peek.go:49-61 peeked */
static int lx_peeked(Lexer *l, const char *token, const char *const *except, int nexcept) {
    if (lx_hasPrefix(l, token)) {
        for (int i = 0; i < nexcept; i++) {
            size_t tl = strlen(token), el = strlen(except[i]);
            char *cat = (char *)malloc(tl + el + 1);
            memcpy(cat, token, tl); memcpy(cat + tl, except[i], el + 1);
            int hit = lx_hasPrefix(l, cat);
            free(cat);
            if (hit) return 0;
        }
        return 1;
    }
    return 0;
}
/* peek.go:65-89 peekedWhitespaced */
static int lx_peekedWhitespaced(Lexer *l, const char *const *tokens, int ntokens) {
    for (int t = 0; t < ntokens; t++) {
        long long i = 0;
        for (;; i++) {
            int32_t *r; int cnt = lx_peekN(l, i + 1, &r);
            (void)cnt; /* Go indexes r[i]; cnt > i always holds here (see DESIGN.md, window analysis) */
            if (r[i] == RUNE_EOF) return 0;
            if (!go_is_space(r[i])) break;
        }
        int32_t *pk; int cnt = lx_peekN(l, i + (long long)strlen(tokens[t]), &pk);
        if (runes_have_prefix(pk + i, cnt - (int)i, tokens[t])) return 1;
    }
    return 0;
}
/* peek.go:100-108 peekedOneOf */
static int lx_peekedOneOf(Lexer *l, const char *runes) {
    for (const char *c = runes; *c; c++) { char tok[2] = { *c, 0 }; if (lx_peeked(l, tok, NULL, 0)) return 1; }
    return 0;
}
/* position.go:68-70 isEmpty */
static int lx_isEmpty(Lexer *l) { return lx_peek(l) == RUNE_EOF; }

/* consume.go:9-13 consume: one next() per RUNE of s */
static void lx_consume_nrunes(Lexer *l, long long nrunes) { for (long long i = 0; i < nrunes; i++) lx_next(l); }
static long long utf8_rune_count(const char *s) {
    size_t n = strlen(s), i = 0; long long c = 0;
    while (i < n) { int w; go_decode_rune((const uint8_t *)s + i, n - i, &w); i += w; c++; }
    return c;
}
static void lx_consume(Lexer *l, const char *s) { lx_consume_nrunes(l, utf8_rune_count(s)); }
/* consume.go:18-32 consumed */
static int lx_consumed(Lexer *l, const char *token, const char *const *except, int nexcept) {
    if (lx_peeked(l, token, except, nexcept)) { lx_consume(l, token); return 1; }
    return 0;
}
/* consume.go:37-47 consumedWhitespaced: consumes l.width RUNES where width is a BYTE count */
static int lx_consumedWhitespaced(Lexer *l, const char *const *tokens, int ntokens) {
    if (lx_peekedWhitespaced(l, tokens, ntokens)) { lx_consume_nrunes(l, l->width); return 1; }
    return 0;
}
/* consume.go:50-61 consumeWhitespace (test-only in the reference) */
static void lx_consumeWhitespace(Lexer *l) {
    for (;;) { int32_t r = lx_next(l); if (!go_is_space(r)) { lx_backup(l); break; } }
}
/* consume.go:65-80 consumeUntil */
static int lx_consumeUntil(Lexer *l, const int32_t *except, int nexcept) {
    int consumed = 0;
    for (;;) {
        int32_t le = lx_next(l);
        if (le == RUNE_EOF) { lx_backup(l); return consumed; }
        for (int i = 0; i < nexcept; i++) if (le == except[i]) { lx_backup(l); return consumed; }
        consumed = 1;
    }
}

/* discard.go:68-71 flush */
static void lx_flush(Lexer *l) { gs_clear(&l->buffer); l->start = l->pos; }
/* discard.go:17-38 discardN */
static void lx_discardN(Lexer *l, long long n) {
    int32_t *rs; int cnt = lx_peekN(l, n, &rs);
    for (int i = 0; i < cnt; i++) {
        int32_t r = rs[i];
        if (r == RUNE_EOF) { lx_flush(l); return; }
        int w = go_rune_len(r);
        w = br_discard(&l->reader, w);
        l->pos.column += w;
        if (r == '\n') resetPosition(l);
    }
    l->start = l->pos;
}
static void lx_discard(Lexer *l) { lx_discardN(l, 1); }
/* discard.go:41-51 discardUntil */
static void lx_discardUntil(Lexer *l, const char *const *tokens, int ntokens) {
    for (;;) {
        for (int t = 0; t < ntokens; t++) if (lx_hasPrefix(l, tokens[t])) return;
        if (lx_isEmpty(l)) return; /* guard: Go would spin at EOF; unreachable from state.go:203 (token was just peeked) */
        lx_discard(l);
    }
}
/* discard.go:55-65 stripWhitespace */
static void lx_stripWhitespace(Lexer *l) {
    for (;;) { int32_t r = lx_peek(l); if (!go_is_space(r)) break; lx_discard(l); }
}

/* emit.go:7-19 emit */
static void lx_emit(Lexer *l, int typ) {
    send(l, typ, l->buffer.p, l->buffer.len, l->start);
    l->lastType = typ;
    gs_clear(&l->lastValue); gs_append(&l->lastValue, l->buffer.p, l->buffer.len);
    gs_clear(&l->buffer);
    l->start = l->pos;
}
/* emit.go:23-32 emitSynthetic */
static void lx_emitSynthetic(Lexer *l, int typ, const char *val) {
    position zero = {0, 0};
    send(l, typ, (const uint8_t *)val, strlen(val), zero);
    l->lastType = typ;
    gs_clear(&l->lastValue); gs_appends(&l->lastValue, val);
}

/* fmt %+v / %d of position */
static void fmt_pos_plus_v(gstr *o, position p) { char t[96]; snprintf(t, sizeof t, "{line:%lld column:%lld}", p.line, p.column); gs_appends(o, t); }
static void fmt_pos_d(gstr *o, position p) { char t[96]; snprintf(t, sizeof t, "{%lld %lld}", p.line, p.column); gs_appends(o, t); }

/* error.go:10-12 context */
static void lx_context(Lexer *l, gstr *ctx) { gs_append(ctx, l->lastValue.p, l->lastValue.len); gs_append(ctx, l->buffer.p, l->buffer.len); }

/* error.go:15-23 errorf / error.go:37-45 warningf share the format "%s at position: %+v, following %q" */
static void lx_send_with_context(Lexer *l, int typ, const uint8_t *msg, size_t msglen) {
    gstr v = {0}, ctx = {0};
    gs_append(&v, msg, msglen);
    gs_appends(&v, " at position: ");
    fmt_pos_plus_v(&v, l->pos);
    gs_appends(&v, ", following ");
    lx_context(l, &ctx);
    go_quote(&v, ctx.p, ctx.len);
    send(l, typ, v.p, v.len, l->pos);
    gs_free(&v); gs_free(&ctx);
}
static state_id lx_errorf_malformed(Lexer *l) { /* state.go:152,173,315: "malformed argument: %s", l.buffer */
    gstr m = {0}; gs_appends(&m, "malformed argument: "); gs_append(&m, l->buffer.p, l->buffer.len);
    lx_send_with_context(l, LexemeError, m.p, m.len); gs_free(&m);
    return ST_NIL;
}
static state_id lx_warningf(Lexer *l, const char *msg) {
    lx_send_with_context(l, LexemeWarning, (const uint8_t *)msg, strlen(msg));
    return ST_lexComment;
}

/* stack.go:7-27 */
static void lx_push(Lexer *l, state_id s) { if (l->nstack < 8) l->stack[l->nstack++] = s; }
static state_id lx_pop(Lexer *l) {
    if (l->nstack == 0) { lx_send_with_context(l, LexemeError, (const uint8_t *)"syntax error", 12); return ST_NIL; }
    return l->stack[--l->nstack];
}
static int lx_emptyStack(Lexer *l) { return l->nstack == 0; }

/* ------------------------------------------------------------------------------------------ */
/* state.go                                                                                    */
/* ------------------------------------------------------------------------------------------ */
static const char *const TOK_COMMENTS[2] = { "//", "#" }; /* golangComment, yamlComment (lexeme.go:41-42) */

/* state.go:15-36 lex */
static state_id st_lex(Lexer *l) {
    lx_stripWhitespace(l);
    if (lx_isEmpty(l)) {
        if (!lx_emptyStack(l)) return lx_pop(l);
        lx_emitSynthetic(l, LexemeEOF, "");
        return ST_NIL;
    }
    if (lx_consumedWhitespaced(l, TOK_COMMENTS, 2)) return ST_lexCommentStart;
    if (lx_consumed(l, "+", NULL, 0)) return ST_lexMarkerStart;
    lx_discard(l);
    return ST_lex;
}
/* state.go:39-43 lexCommentStart */
static state_id st_lexCommentStart(Lexer *l) { lx_emit(l, LexemeComment); return ST_lexComment; }
/* state.go:46-57 lexComment */
static state_id st_lexComment(Lexer *l) {
    if (lx_consumed(l, "+", NULL, 0)) return ST_lexMarkerStart;
    if (lx_peeked(l, "\n", NULL, 0) || lx_isEmpty(l)) return ST_lex;
    lx_discard(l);
    return ST_lexComment;
}
/* state.go:60-68 lexMarkerStart */
static state_id st_lexMarkerStart(Lexer *l) {
    if (go_is_letter(lx_peek(l))) { lx_emit(l, LexemeMarkerStart); return ST_lexMarker; }
    return ST_lexComment;
}
static const int32_t EXC_NAME[16] = { ':', '=', ' ', '"', '\'', '`', ',', '+', '{', '}', '[', ']', '(', ')', ';', '\n' };
static const int32_t EXC_NAKED[15] = { ':', '=', ' ', '"', '\'', '`', ',', '+', '{', '}', '[', ']', '(', ')', '\n' };

/* state.go:71-116 lexMarker */
static state_id st_lexMarker(Lexer *l) {
    if (!lx_consumeUntil(l, EXC_NAME, 16)) { lx_backup(l); lx_flush(l); return ST_lexComment; }
    if (lx_peeked(l, ":", NULL, 0)) {
        lx_emit(l, LexemeScope);
        lx_consume(l, ":");
        lx_emit(l, LexemeSeparator);
        return ST_lexMarker;
    }
    if (lx_peeked(l, " ", NULL, 0) || lx_peeked(l, "\n", NULL, 0) || lx_peek(l) == RUNE_EOF) {
        if (l->lastType != LexemeSeparator) return lx_warningf(l, "marker without scope found");
        lx_emit(l, LexemeArg);
        lx_emitSynthetic(l, LexemeSyntheticBoolLiteral, "true");
        lx_emitSynthetic(l, LexemeMarkerEnd, "\n");
        return ST_lexComment;
    }
    if (lx_peeked(l, "=", NULL, 0)) {
        if (l->lastType != LexemeSeparator) return lx_warningf(l, "marker without scope found");
        lx_emit(l, LexemeArg);
        lx_consume(l, "=");
        lx_emit(l, LexemeArgAssignment);
        return ST_lexArgValueInitial;
    }
    return lx_warningf(l, "invalid marker found");
}
/* state.go:118-154 lexArgs */
static state_id st_lexArgs(Lexer *l) {
    if (!lx_consumeUntil(l, EXC_NAME, 16)) {
        lx_backup(l); lx_flush(l);
        lx_emitSynthetic(l, LexemeMarkerEnd, "\n");
        return ST_lex;
    }
    lx_emit(l, LexemeArg);
    if (lx_consumed(l, "=", NULL, 0)) { lx_emit(l, LexemeArgAssignment); return ST_lexArgValueInitial; }
    if (lx_peeked(l, " ", NULL, 0) || lx_peeked(l, "\n", NULL, 0) || lx_peek(l) == RUNE_EOF) {
        lx_emitSynthetic(l, LexemeSyntheticBoolLiteral, "true");
        lx_emitSynthetic(l, LexemeMarkerEnd, "\n");
        return ST_lexComment;
    }
    if (lx_peeked(l, ",", NULL, 0)) { lx_emitSynthetic(l, LexemeSyntheticBoolLiteral, "true"); return ST_lexMoreArgs; }
    return lx_errorf_malformed(l);
}

/* state.go:193-194,199,209: rawErrorf(`unmatched string delimiter %s at position %+v, following %q`, quote, pos, context) */
static state_id lx_unmatched(Lexer *l, const char *quote, position pos, const gstr *context) {
    gstr v = {0};
    gs_appends(&v, "unmatched string delimiter "); gs_appends(&v, quote);
    gs_appends(&v, " at position "); fmt_pos_plus_v(&v, pos);
    gs_appends(&v, ", following "); go_quote(&v, context->p, context->len);
    send(l, LexemeError, v.p, v.len, l->pos);
    gs_free(&v);
    return ST_NIL;
}
/* state.go:176-221 lexStringLiteral; returns 1 if "present" and sets *next */
static int st_lexStringLiteral(Lexer *l, state_id nextState, state_id *next) {
    const char *quote;
    int32_t p = lx_peek(l);
    if (p == '\'') quote = "'"; else if (p == '"') quote = "\""; else if (p == '`') quote = "`"; else return 0;
    lx_consume(l, quote);
    lx_emit(l, LexemeQuote);
    position pos = l->pos;
    gstr context = {0}; lx_context(l, &context);
    for (;;) {
        if (lx_peek(l) == RUNE_EOF) { *next = lx_unmatched(l, quote, pos, &context); gs_free(&context); return 1; }
        if (lx_peeked(l, "\n", NULL, 0)) {
            if (quote[0] == '`') {
                lx_next(l);
                if (lx_peekedWhitespaced(l, TOK_COMMENTS, 2)) { lx_discardUntil(l, TOK_COMMENTS, 2); lx_discard(l); }
            } else { *next = lx_unmatched(l, quote, pos, &context); gs_free(&context); return 1; }
        } else if (lx_peeked(l, quote, NULL, 0)) {
            lx_emit(l, LexemeStringLiteral);
            lx_consume(l, quote);
            lx_emit(l, LexemeQuote);
            gs_free(&context);
            *next = nextState; return 1;
        } else {
            lx_next(l);
        }
    }
}
/* state.go:223-252 lexNumericLiteral */
static int st_lexNumericLiteral(Lexer *l, state_id nextState, state_id *next) {
    int32_t n = lx_peek(l);
    if (lx_peekedOneOf(l, ".-") || go_is_number(lx_peek(l))) {
        int isfloat = n == '.';
        for (;;) {
            lx_next(l);
            if (lx_peekedOneOf(l, ".eE-")) { isfloat = 1; continue; }
            if (!go_is_number(lx_peek(l))) break;
        }
        lx_push(l, nextState);
        *next = isfloat ? ST_lexFloatLiteral : ST_lexIntegerLiteral;
        return 1;
    }
    return 0;
}
static const char *strconv_err_text(int code) { return code == 2 ? "value out of range" : "invalid syntax"; }
/* state.go:254-265 / 267-276: rawErrorf("invalid float literal %q: %s before position %d", value, err, pos) */
static state_id lx_numeric_error(Lexer *l, const char *kind, const char *fn, int code) {
    gstr v = {0};
    gs_appends(&v, "invalid "); gs_appends(&v, kind); gs_appends(&v, " literal ");
    go_quote(&v, l->buffer.p, l->buffer.len);
    gs_appends(&v, ": strconv."); gs_appends(&v, fn); gs_appends(&v, ": parsing ");
    go_quote(&v, l->buffer.p, l->buffer.len);
    gs_appends(&v, ": "); gs_appends(&v, strconv_err_text(code));
    gs_appends(&v, " before position "); fmt_pos_d(&v, l->pos);
    send(l, LexemeError, v.p, v.len, l->pos);
    gs_free(&v);
    return ST_NIL;
}
static state_id st_lexFloatLiteral(Lexer *l) {
    int code = go_parse_float_err(l->buffer.p, l->buffer.len);
    if (code) return lx_numeric_error(l, "float", "ParseFloat", code);
    lx_emit(l, LexemeFloatLiteral);
    return lx_pop(l);
}
static state_id st_lexIntegerLiteral(Lexer *l) {
    int code = go_atoi_err(l->buffer.p, l->buffer.len);
    if (code) return lx_numeric_error(l, "integer", "Atoi", code);
    lx_emit(l, LexemeIntegerLiteral);
    return lx_pop(l);
}
/* state.go:278-286 lexBooleanLiteral */
static int st_lexBooleanLiteral(Lexer *l, state_id nextState, state_id *next) {
    static const char *const T[1] = { "true" }; static const char *const F[1] = { "false" };
    if (lx_consumedWhitespaced(l, T, 1) || lx_consumedWhitespaced(l, F, 1)) { lx_emit(l, LexemeBoolLiteral); *next = nextState; return 1; }
    return 0;
}
/* state.go:288-302 lexNakedStringLiteral */
static int st_lexNakedStringLiteral(Lexer *l, state_id nextState, state_id *next) {
    if (!lx_consumeUntil(l, EXC_NAKED, 15)) return 0;
    lx_emit(l, LexemeStringLiteral);
    *next = nextState; return 1;
}
/* state.go:156-174 lexArgValueInitial */
static state_id st_lexArgValueInitial(Lexer *l) {
    state_id nx;
    if (st_lexStringLiteral(l, ST_lexMoreArgs, &nx)) return nx;
    if (st_lexNumericLiteral(l, ST_lexMoreArgs, &nx)) return nx;
    if (st_lexBooleanLiteral(l, ST_lexMoreArgs, &nx)) return nx;
    if (st_lexNakedStringLiteral(l, ST_lexMoreArgs, &nx)) return nx;
    return lx_errorf_malformed(l);
}
/* state.go:304-317 lexMoreArgs */
static state_id st_lexMoreArgs(Lexer *l) {
    if (lx_consumed(l, ",", NULL, 0)) { lx_emit(l, LexemeArgDelimiter); return ST_lexArgs; }
    if (lx_peeked(l, " ", NULL, 0) || lx_peeked(l, "\n", NULL, 0) || lx_peek(l) == RUNE_EOF) {
        lx_emitSynthetic(l, LexemeMarkerEnd, "\n");
        return ST_lexComment;
    }
    return lx_errorf_malformed(l);
}

/* lexer.go:43-48 Run */
static void lexer_run(Lexer *l) {
    state_id st = ST_lex;
    while (st != ST_NIL) {
        switch (st) {
        case ST_lex: st = st_lex(l); break;
        case ST_lexCommentStart: st = st_lexCommentStart(l); break;
        case ST_lexComment: st = st_lexComment(l); break;
        case ST_lexMarkerStart: st = st_lexMarkerStart(l); break;
        case ST_lexMarker: st = st_lexMarker(l); break;
        case ST_lexArgs: st = st_lexArgs(l); break;
        case ST_lexArgValueInitial: st = st_lexArgValueInitial(l); break;
        case ST_lexFloatLiteral: st = st_lexFloatLiteral(l); break;
        case ST_lexIntegerLiteral: st = st_lexIntegerLiteral(l); break;
        case ST_lexMoreArgs: st = st_lexMoreArgs(l); break;
        default: st = ST_NIL;
        }
    }
}

/* ------------------------------------------------------------------------------------------ */
/* exported test / baseline API                                                                */
/* ------------------------------------------------------------------------------------------ */

/* Lex one document; *out receives a malloc'd serialised lexeme stream (see `sink`). */
int obo_lex(const uint8_t *doc, uint64_t n, uint8_t **out, uint64_t *outlen, uint64_t *n_lexemes) {
    sink s; memset(&s, 0, sizeof s); s.mode = 0;
    Lexer l; lexer_init(&l, doc, (size_t)n, &s);
    lexer_run(&l);
    lexer_free(&l);
    *out = s.out.p; *outlen = s.out.len; if (n_lexemes) *n_lexemes = s.n_lexemes;
    return 0;
}
void obo_free(void *p) { free(p); }

/* Lex a packed batch serially; the per-document streams are concatenated, doc_stream_off[ndocs+1]
 * receives the byte offset of each document's stream, doc_lexemes[ndocs] its lexeme count. */
int obo_lex_batch(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, uint8_t **out, uint64_t *outlen,
                  uint64_t *doc_stream_off, uint64_t *doc_lexemes) {
    sink s; memset(&s, 0, sizeof s); s.mode = 0;
    for (uint32_t d = 0; d < ndocs; d++) {
        if (doc_stream_off) doc_stream_off[d] = s.out.len;
        uint64_t before = s.n_lexemes;
        Lexer l; lexer_init(&l, bytes + doc_off[d], (size_t)(doc_off[d + 1] - doc_off[d]), &s);
        lexer_run(&l);
        lexer_free(&l);
        if (doc_lexemes) doc_lexemes[d] = s.n_lexemes - before;
    }
    if (doc_stream_off) doc_stream_off[ndocs] = s.out.len;
    *out = s.out.p; *outlen = s.out.len;
    return 0;
}

/* CPU baseline: count + hash only, documents statically partitioned over nthreads pthreads. */
typedef struct { const uint8_t *bytes; const uint64_t *doc_off; uint32_t d0, d1; uint64_t n_lexemes, n_markers, hash; uint64_t *doc_hash; } scan_job;
static void *scan_worker(void *arg) {
    scan_job *j = (scan_job *)arg;
    for (uint32_t d = j->d0; d < j->d1; d++) {
        sink s; memset(&s, 0, sizeof s); s.mode = 1; s.hash = 0xcbf29ce484222325ULL;
        Lexer l; lexer_init(&l, j->bytes + j->doc_off[d], (size_t)(j->doc_off[d + 1] - j->doc_off[d]), &s);
        lexer_run(&l);
        lexer_free(&l);
        j->n_lexemes += s.n_lexemes; j->n_markers += s.n_markers; j->hash ^= s.hash * (2 * (uint64_t)d + 1);
        if (j->doc_hash) j->doc_hash[d] = s.hash;
    }
    return NULL;
}
int obo_scan_batch(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, int nthreads,
                   uint64_t *n_lexemes, uint64_t *n_markers, uint64_t *hash, uint64_t *doc_hash) {
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    scan_job jobs[256]; pthread_t th[256];
    for (int t = 0; t < nthreads; t++) {
        memset(&jobs[t], 0, sizeof jobs[t]);
        jobs[t].bytes = bytes; jobs[t].doc_off = doc_off; jobs[t].doc_hash = doc_hash;
        jobs[t].d0 = (uint32_t)((uint64_t)ndocs * t / nthreads);
        jobs[t].d1 = (uint32_t)((uint64_t)ndocs * (t + 1) / nthreads);
        if (nthreads == 1) scan_worker(&jobs[t]); else pthread_create(&th[t], NULL, scan_worker, &jobs[t]);
    }
    uint64_t nl = 0, nm = 0, h = 0;
    for (int t = 0; t < nthreads; t++) {
        if (nthreads > 1) pthread_join(th[t], NULL);
        nl += jobs[t].n_lexemes; nm += jobs[t].n_markers; h ^= jobs[t].hash;
    }
    if (n_lexemes) *n_lexemes = nl;
    if (n_markers) *n_markers = nm;
    if (hash) *hash = h;
    return 0;
}

/* ---- primitive hooks for the reference's white-box tests (consume/peek _internal_test.go) ---- */
typedef struct { Lexer l; sink s; uint8_t *copy; } prim;
void *obo_prim_new(const uint8_t *doc, uint64_t n) {
    prim *p = (prim *)calloc(1, sizeof *p);
    p->copy = (uint8_t *)malloc(n ? n : 1); memcpy(p->copy, doc, n);
    p->s.mode = 0;
    lexer_init(&p->l, p->copy, (size_t)n, &p->s);
    return p;
}
void obo_prim_free(void *h) { prim *p = (prim *)h; lexer_free(&p->l); gs_free(&p->s.out); free(p->copy); free(p); }
void obo_prim_consume(void *h, const char *s) { lx_consume(&((prim *)h)->l, s); }
int obo_prim_consumed(void *h, const char *tok, const char *const *exc, int nexc) { return lx_consumed(&((prim *)h)->l, tok, exc, nexc); }
int obo_prim_consumedWhitespaced(void *h, const char *const *toks, int n) { return lx_consumedWhitespaced(&((prim *)h)->l, toks, n); }
void obo_prim_consumeWhitespace(void *h) { lx_consumeWhitespace(&((prim *)h)->l); }
int obo_prim_consumeUntil(void *h, const int32_t *exc, int n) { return lx_consumeUntil(&((prim *)h)->l, exc, n); }
int32_t obo_prim_peek(void *h) { return lx_peek(&((prim *)h)->l); }
int obo_prim_peekN(void *h, int n, int32_t *out) { int32_t *rs; int c = lx_peekN(&((prim *)h)->l, n, &rs); memcpy(out, rs, (size_t)c * sizeof(int32_t)); return c; }
int obo_prim_peeked(void *h, const char *tok, const char *const *exc, int nexc) { return lx_peeked(&((prim *)h)->l, tok, exc, nexc); }
int obo_prim_peekedWhitespaced(void *h, const char *const *toks, int n) { return lx_peekedWhitespaced(&((prim *)h)->l, toks, n); }
uint64_t obo_prim_buffer(void *h, uint8_t *out, uint64_t cap) { prim *p = (prim *)h; uint64_t n = p->l.buffer.len < cap ? p->l.buffer.len : cap; memcpy(out, p->l.buffer.p, n); return p->l.buffer.len; }
void obo_prim_pos(void *h, int64_t *line, int64_t *col) { prim *p = (prim *)h; *line = p->l.pos.line; *col = p->l.pos.column; }

/* strconv helpers exposed so tests can cross-check them against Python's float()/int() */
int obo_parse_float_err(const uint8_t *s, uint64_t n) { return go_parse_float_err(s, (size_t)n); }
int obo_atoi_err(const uint8_t *s, uint64_t n) { return go_atoi_err(s, (size_t)n); }
uint64_t obo_quote(const uint8_t *s, uint64_t n, uint8_t *out, uint64_t cap) {
    gstr o = {0}; go_quote(&o, s, (size_t)n);
    uint64_t len = o.len; memcpy(out, o.p, len < cap ? len : cap); gs_free(&o); return len;
}
/* out[i] bit 0: unicode.IsLetter, bit 1: IsNumber, bit 2: IsSpace, bit 3: strconv.IsPrint of cps[i] */
void obo_classify(const int32_t *cps, uint64_t n, uint8_t *out) {
    for (uint64_t i = 0; i < n; i++) {
        int32_t r = cps[i];
        out[i] = (uint8_t)(go_is_letter(r) | go_is_number(r) << 1 | go_is_space(r) << 2 | go_is_print(r) << 3);
    }
}
