/*
 * obm_core.h -- the exact marker lexer as straight-line code over an in-memory document, emitting
 * the canonical tuple stream defined in include/obmarkers.h.
 *
 * Compiled for the device by nvcc (used by every kernel in obm_lib.cu) and, for logic tests
 * only, for the host by g++ (tests/hostsim).  It is NOT a CPU fallback: libobmarkers.so exports no
 * host lexing entry point.
 *
 * What it restates (reference: internal/markers/lexer @ 2827f233):
 *   state machine            state.go:15-317   (lex, lexComment, lexMarkerStart, lexMarker, lexArgs,
 *                                               lexArgValueInitial + literal lexers, lexMoreArgs)
 *   next/backup/positions    position.go:18-65
 *   peek windows             peek.go:20-96 over bufio.Reader (default 4096-byte buffer, lexer.go:38)
 *   discard / flush          discard.go:17-71
 *   emit / emitSynthetic     emit.go:7-32
 * Because the document is resident in memory, bufio.Reader.Peek(n) is the closed form
 * "min(n, 4096, remaining) bytes at the read offset" (DESIGN.md, "peek window").
 *
 * The reference's `buffer` string is represented implicitly: un-emitted text is doc[s, p) plus the
 * PART tuples already sent; `start` is the offset s.  See obmarkers.h for the pseudo-tuples.
 */
#ifndef OBM_CORE_H
#define OBM_CORE_H

#include <stdint.h>
#include "../../include/obmarkers.h"

#if defined(__CUDACC__)
#define OBM_HD __host__ __device__ __forceinline__
#define OBM_FN __host__ __device__ inline
#define OBM_HD_NOINLINE __host__ __device__ __noinline__
/* hides a value from the optimiser: keeps the state variable of the line machine a run-time value so that
 * the compiler cannot thread jumps from one state's code straight into the next (which would leave the
 * lanes of a warp in different copies of the loop body and never reconverged) */
#if defined(__CUDA_ARCH__)
#define OBM_OPAQUE(x) asm volatile("" : "+r"(x))
#else
#define OBM_OPAQUE(x) ((void)0)
#endif
#else
#define OBM_HD inline
#define OBM_FN inline
#define OBM_HD_NOINLINE inline
#define OBM_OPAQUE(x) ((void)0)
#endif

namespace obm {

/* Range tables + constants reachable from both host and device builds. */
struct Tables {
    const unsigned int (*letter)[2]; int n_letter;
    const unsigned int (*number)[2]; int n_number;
    const char *f64_overflow_digits; /* decimal digits of 2^1024 - 2^970 (309 of them) */
};

enum { RUNE_ERR = 0xFFFD, RUNE_EOF = -1 };
enum { BUFIO_WINDOW = 4096 }; /* bufio.defaultBufSize, lexer.go:38 */

/* utf8.DecodeRune over doc[at, lim) */
OBM_HD int decode_rune(const uint8_t *d, uint32_t at, uint32_t lim, uint32_t &w) {
    if (at >= lim) { w = 0; return RUNE_EOF; }
    uint32_t c0 = d[at];
    if (c0 < 0x80) { w = 1; return (int)c0; }
    w = 1;
    if (c0 < 0xC2 || c0 > 0xF4) return RUNE_ERR;
    uint32_t avail = lim - at;
    if (c0 < 0xE0) {
        if (avail < 2 || (d[at + 1] & 0xC0) != 0x80) return RUNE_ERR;
        w = 2; return (int)(((c0 & 0x1F) << 6) | (d[at + 1] & 0x3Fu));
    }
    if (c0 < 0xF0) {
        uint32_t lo = 0x80, hi = 0xBF;
        if (c0 == 0xE0) lo = 0xA0; else if (c0 == 0xED) hi = 0x9F;
        if (avail < 3) return RUNE_ERR;
        uint32_t c1 = d[at + 1], c2 = d[at + 2];
        if (c1 < lo || c1 > hi || (c2 & 0xC0) != 0x80) return RUNE_ERR;
        w = 3; return (int)(((c0 & 0x0F) << 12) | ((c1 & 0x3F) << 6) | (c2 & 0x3F));
    }
    {
        uint32_t lo = 0x80, hi = 0xBF;
        if (c0 == 0xF0) lo = 0x90; else if (c0 == 0xF4) hi = 0x8F;
        if (avail < 4) return RUNE_ERR;
        uint32_t c1 = d[at + 1], c2 = d[at + 2], c3 = d[at + 3];
        if (c1 < lo || c1 > hi || (c2 & 0xC0) != 0x80 || (c3 & 0xC0) != 0x80) return RUNE_ERR;
        w = 4; return (int)(((c0 & 0x07) << 18) | ((c1 & 0x3F) << 12) | ((c2 & 0x3F) << 6) | (c3 & 0x3F));
    }
}

OBM_HD bool in_ranges(const unsigned int (*t)[2], int n, int r) {
    int lo = 0, hi = n - 1;
    while (lo <= hi) {
        int mid = (lo + hi) >> 1;
        if ((unsigned)r < t[mid][0]) hi = mid - 1;
        else if ((unsigned)r > t[mid][1]) lo = mid + 1;
        else return true;
    }
    return false;
}
/* unicode.IsSpace (White_Space) */
OBM_HD bool is_space(int r) {
    if (r < 0) return false;
    if (r < 0x80) return r == ' ' || (r >= 0x09 && r <= 0x0D);
    if (r <= 0xFF) return r == 0x85 || r == 0xA0;
    return r == 0x1680 || (r >= 0x2000 && r <= 0x200A) || r == 0x2028 || r == 0x2029 || r == 0x202F || r == 0x205F || r == 0x3000;
}
OBM_HD bool is_letter(const Tables &T, int r) {
    if (r < 0) return false;
    if (r < 0x80) { unsigned c = (unsigned)r | 0x20u; return c >= 'a' && c <= 'z'; }
    return in_ranges(T.letter, T.n_letter, r);
}
OBM_HD bool is_letter_ascii(int r) { unsigned c = (unsigned)r | 0x20u; return r >= 0 && r < 0x80 && c >= 'a' && c <= 'z'; }
OBM_HD bool is_digit_ascii(int r) { return r >= '0' && r <= '9'; }
OBM_HD bool is_number(const Tables &T, int r) {
    if (r < 0) return false;
    if (r < 0x80) return r >= '0' && r <= '9';
    return in_ranges(T.number, T.n_number, r);
}

/* Delimiter sets of consumeUntil (state.go:72-76, 119-123, 289-293) as 128-bit ASCII masks.
 * name set:  : = SP " ' ` , + { } [ ] ( ) ; \n      naked-value set: the same without ';' */
OBM_HD bool is_name_delim(uint32_t c) {
    /* 128-bit membership mask, one 32-bit word per 32 code points:
     * word0: \n(10)   word1: SP(32) "(34) '(39) ((40) )(41) +(43) ,(44) :(58) ;(59) =(61)
     * word2: [(91) ](93)   word3: `(96) {(123) }(125) */
    const uint32_t m0 = 1u << 10;
    const uint32_t m1 = (1u << 0) | (1u << 2) | (1u << 7) | (1u << 8) | (1u << 9) | (1u << 11) | (1u << 12) | (1u << 26) | (1u << 27) | (1u << 29);
    const uint32_t m2 = (1u << (91 - 64)) | (1u << (93 - 64));
    const uint32_t m3 = (1u << 0) | (1u << (123 - 96)) | (1u << (125 - 96));
    /* letters, digits and '.', '-', '_', '/' (what names are made of) leave through the first test */
    uint32_t lo = (c & 0x40u) ? ((c & 0x20u) ? m3 : m2) : ((c & 0x20u) ? m1 : m0);
    return c < 0x80u && ((lo >> (c & 31u)) & 1u);
}
OBM_HD bool is_naked_delim(uint32_t c) { return c != ';' && is_name_delim(c); }

/* strconv.ParseFloat(s, 64) error class: 0 ok, 1 invalid syntax, 2 value out of range (state.go:258).
 * Restated from Go 1.16 strconv/atof.go (special, readFloat) for decimal input; see oracle notes. */
OBM_HD_NOINLINE int parse_float_err(const Tables &T, const uint8_t *s, uint32_t n) {
    if (n == 0) return 1;
    uint32_t i = 0;
    {
        uint32_t j = 0; uint32_t c0 = s[0];
        if (c0 == '+' || c0 == '-') j = 1;
        if (j < n && (j == 1 || (c0 | 0x20) == 'i')) {
            const char inf[9] = {'i', 'n', 'f', 'i', 'n', 'i', 't', 'y', 0};
            uint32_t k = 0;
            while (j + k < n && k < 8 && (uint32_t)(s[j + k] | 0x20) == (uint32_t)inf[k]) k++;
            if (k > 3 && k < 8) k = 3;
            if (k == 3 || k == 8) return (j + k == n) ? 0 : 1;
        } else if ((c0 | 0x20) == 'n') {
            if (n >= 3 && (s[1] | 0x20) == 'a' && (s[2] | 0x20) == 'n') return n == 3 ? 0 : 1;
        }
    }
    if (s[i] == '+' || s[i] == '-') i++;
    if (i + 2 < n && s[i] == '0' && (s[i + 1] | 0x20) == 'x') return 1; /* hex floats: unreachable from the lexer's alphabet */
    bool sawdot = false, sawdigits = false, nonzero = false;
    long long nd = 0, dp = 0;
    uint32_t dbeg = i;
    for (; i < n; i++) {
        uint32_t c = s[i];
        if (c == '_') return 1; /* underscores need a base prefix */
        if (c == '.') { if (sawdot) break; sawdot = true; dp = nd; continue; }
        if (c >= '0' && c <= '9') {
            sawdigits = true;
            if (c == '0' && nd == 0) { dp--; continue; }
            nd++; nonzero = true; continue;
        }
        break;
    }
    uint32_t dend = i;
    if (!sawdigits) return 1;
    if (!sawdot) dp = nd;
    if (i < n && (s[i] | 0x20) == 'e') {
        i++;
        if (i >= n) return 1;
        int esign = 1;
        if (s[i] == '+') i++; else if (s[i] == '-') { i++; esign = -1; }
        if (i >= n || s[i] < '0' || s[i] > '9') return 1;
        long long e = 0;
        for (; i < n && ((s[i] >= '0' && s[i] <= '9') || s[i] == '_'); i++) {
            if (s[i] == '_') return 1;
            if (e < 10000) e = e * 10 + (s[i] - '0');
        }
        dp += e * esign;
    }
    if (i != n) return 1;
    if (!nonzero) return 0;
    if (dp > 309) return 2;
    if (dp < 309) return 0;
    uint32_t k = 0; bool started = false;
    for (uint32_t j = dbeg; j < dend; j++) {
        uint32_t c = s[j];
        if (c == '.') continue;
        if (!started) { if (c == '0') continue; started = true; }
        if (k < 309) {
            uint32_t t = (uint32_t)T.f64_overflow_digits[k];
            if (c > t) return 2;
            if (c < t) return 0;
            k++;
        } else return 2;
    }
    for (; k < 309; k++) if (T.f64_overflow_digits[k] != '0') return 0;
    return 2;
}

/* strconv.Atoi error class (state.go:269); int is 64-bit; overflow is reported when it happens. */
OBM_HD_NOINLINE int atoi_err(const uint8_t *s, uint32_t n) {
    uint32_t i = 0; bool neg = false;
    if (n == 0) return 1;
    if (s[0] == '+' || s[0] == '-') { neg = s[0] == '-'; i = 1; }
    if (i >= n) return 1;
    const uint64_t cutoff = 0xFFFFFFFFFFFFFFFFull / 10 + 1;
    uint64_t v = 0;
    for (; i < n; i++) {
        if (s[i] < '0' || s[i] > '9') return 1;
        if (v >= cutoff) return 2;
        v *= 10;
        uint64_t v1 = v + (uint64_t)(s[i] - '0');
        if (v1 < v) return 2;
        v = v1;
    }
    if (!neg && v >= (1ull << 63)) return 2;
    if (neg && v > (1ull << 63)) return 2;
    return 0;
}

/* ---- sinks ---------------------------------------------------------------------------------- */
struct CountSink {
    uint64_t n_tuples = 0; uint32_t n_markers = 0; uint32_t n_lexemes = 0;
    OBM_HD void put(uint32_t kind, uint32_t off, uint32_t len) {
        (void)off; (void)len;
        n_tuples++;
        n_markers += (kind == OBM_K_MARKER_START);
        n_lexemes += (kind <= OBM_K_EOF) || (kind >= OBM_K_WARN_NOSCOPE);
    }
};
struct WriteSink {
    obm_tuple *out; uint64_t cap; /* tuples beyond cap are dropped (caller detects via count) */
    uint64_t n_tuples = 0; uint32_t n_markers = 0; uint32_t n_lexemes = 0;
    OBM_HD WriteSink(obm_tuple *o, uint64_t c) : out(o), cap(c) {}
    OBM_HD void put(uint32_t kind, uint32_t off, uint32_t len) {
        if (n_tuples < cap) out[n_tuples] = OBM_TUPLE(kind, off, len);
        n_tuples++;
        n_markers += (kind == OBM_K_MARKER_START);
        n_lexemes += (kind <= OBM_K_EOF) || (kind >= OBM_K_WARN_NOSCOPE);
    }
};

/* 32-bit sink for bounded documents (tile path): counts always, writes while n < cap (cap 0 = count only) */
struct SmallSink {
    obm_tuple *out; uint32_t cap; uint32_t n_tuples, n_markers, n_lexemes;
    OBM_HD SmallSink(obm_tuple *o, uint32_t c) : out(o), cap(c), n_tuples(0), n_markers(0), n_lexemes(0) {}
    OBM_HD void put(uint32_t kind, uint32_t off, uint32_t len) {
        if (n_tuples < cap) out[n_tuples] = OBM_TUPLE(kind, off, len);
        n_tuples++;
        n_markers += (kind == OBM_K_MARKER_START);
        n_lexemes += (kind - (uint32_t)OBM_K_PART) > 4u; /* everything but PART, FLUSH, DRIFT, LINE, LINEHI (21..25) */
    }
};

enum RunStatus { RUN_EOF = 0, RUN_LINE_END = 1, RUN_FATAL = 2 };
enum TopState { TOP_LEX = 0, TOP_COMMENT = 1, TOP_FATAL = 2 };

/* Scan accelerator hook: next_interesting(p) returns the smallest q >= p such that doc[q] may be a
 * newline or one of # + / ' (or n).  The exact path uses NoAccel (q = p: no skipping); the tile path
 * answers from its newline/special bitmaps.  Only valid for all-ASCII documents. */
struct NoAccel {
    OBM_HD uint32_t next_interesting(uint32_t p) const { return p; }
};

/* ASCII = true: the caller guarantees every byte of the document is < 0x80 (tile path); rune decoding,
 * the Unicode tables and the U+FFFD over-discard drop out at compile time.
 * SHORT = true: the lexer only sees documents of at most 16 KiB (the tile, pipeline and warp kernels), so no
 * slice can reach OBM_MAX_LEN.  Lexers that may see larger documents (the exact path, the chunk-parallel
 * large path) keep SHORT = false and send every long slice as PART pieces. */

/* peek.go:65-89 for one ASCII token `tok[0..t)` at offset p of doc d[0..n): on success returns true and
 * sets `width` (= l.width after the final peekN: whitespace BYTES + token bytes). */
template <bool ASCII>
OBM_HD_NOINLINE bool peeked_whitespaced_at(const uint8_t *d, uint32_t n, uint32_t p, const char *tok, uint32_t t, uint32_t &width) {
    uint32_t lim = (n - p > (uint32_t)BUFIO_WINDOW) ? p + (uint32_t)BUFIO_WINDOW : n;
    uint32_t o = p;
    for (;;) {
        uint32_t w; int r;
        if (ASCII) { if (o < lim) { r = (int)d[o]; w = 1; } else { r = RUNE_EOF; w = 0; } }
        else r = decode_rune(d, o, lim, w);
        if (r == RUNE_EOF) return false; /* r[i] == eof (real end of input or end of the 4096-byte window) */
        if (!is_space(r)) break;
        o += w;
    }
    if (o + t > lim) return false;
    for (uint32_t k = 0; k < t; k++) if (d[o + k] != (uint8_t)tok[k]) return false;
    width = (o - p) + t;
    return true;
}

/* ---- byte source of a lexer -------------------------------------------------------------------------
 * Default: a plain pointer.  On the device K2 also uses ShBytes: the document bytes it may touch sit in a
 * shared-memory copy, addressed through the 32-bit shared window so that loads are LDS (short scoreboard)
 * instead of generic-address loads; `g` is the equivalent generic pointer for the cold helpers. */
OBM_HD uint32_t src_mis(const uint8_t *d, uint32_t q) { return (uint32_t)((uintptr_t)(d + q) & 3u); }
OBM_HD uint32_t src_ldw(const uint8_t *d, int32_t off) { return *reinterpret_cast<const uint32_t *>(d + off); }
OBM_HD const uint8_t *src_raw(const uint8_t *d) { return d; }
OBM_HD const uint8_t *src_add(const uint8_t *d, uint32_t off) { return d + off; }
struct Quad { uint32_t w[4]; };
OBM_HD Quad src_ldq(const uint8_t *d, uint32_t off16) { /* 16 bytes at a 16-byte aligned offset of a 16-byte aligned base */
    const uint32_t *q = reinterpret_cast<const uint32_t *>(d + off16);
    return Quad{{q[0], q[1], q[2], q[3]}};
}
#if defined(__CUDACC__)
struct ShBytes {
    uint32_t sh; const uint8_t *g;
    __device__ __forceinline__ uint32_t operator[](uint32_t i) const { uint32_t v; asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(sh + i)); return v; }
};
__device__ __forceinline__ uint32_t src_mis(const ShBytes &d, uint32_t q) { return (d.sh + q) & 3u; }
__device__ __forceinline__ uint32_t src_ldw(const ShBytes &d, int32_t off) { uint32_t v; asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(d.sh + (uint32_t)off)); return v; }
__device__ __forceinline__ const uint8_t *src_raw(const ShBytes &d) { return d.g; }
__device__ __forceinline__ ShBytes src_add(const ShBytes &d, uint32_t off) { return ShBytes{d.sh + off, d.g + off}; }
__device__ __forceinline__ Quad src_ldq(const ShBytes &d, uint32_t off16) {
    Quad q;
    asm("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(q.w[0]), "=r"(q.w[1]), "=r"(q.w[2]), "=r"(q.w[3]) : "r"(d.sh + off16));
    return q;
}
#endif

template <class Sink, class Accel = NoAccel, bool ASCII = false, class Src = const uint8_t *, bool SHORT = false>
struct Lexer {
    const Tables &T;
    Src d; uint32_t n;
    uint32_t p, s;                      /* read offset; `start` offset */
    uint32_t line_p, base_p, drift_p;   /* l.pos   == {line_p, p - base_p + 1 - drift_p} */
    uint32_t line_s, base_s;            /* l.start == {line_s, s - base_s + 1 - (drift of that line)} */
    uint32_t line_e, base_e;            /* basis announced by the last LINE tuple */
    uint32_t sv_line, sv_base, sv_drift;/* basis before the '\n' just read by next(), for backup() */
    uint32_t last_w; int last_r;        /* l.width / rune of the last next() */
    uint32_t last_type;                 /* l.lastEmittedLexeme.Type */
    Sink &out;
    Accel accel;
    int32_t wbase; uint32_t wm0, wm1, wm2, wm3; /* ASCII only: cached 128 bytes of "not a letter" bits from wbase */

    /* A lexer instance begins at byte `start_off` of line `first_line`, whose first byte is at
     * `line_base` (document start: 0, 1, 0).  `announce_first`: the first located tuple must be
     * preceded by a LINE tuple (true for every line-mode instance except the document's first line). */
    OBM_HD Lexer(const Tables &t, Src doc, uint32_t len, Sink &sink, uint32_t start_off = 0,
                 uint32_t first_line = 1, uint32_t line_base = 0, bool announce_first = false, Accel acc = Accel())
        : T(t), d(doc), n(len), p(start_off), s(start_off), line_p(first_line), base_p(line_base), drift_p(0),
          line_s(first_line), base_s(line_base), line_e(announce_first ? 0u : 1u), base_e(0),
          sv_line(first_line), sv_base(line_base), sv_drift(0), last_w(0), last_r(RUNE_EOF), last_type(0), out(sink), accel(acc),
          wbase(-0x40000000), wm0(0), wm1(0), wm2(0), wm3(0) {}

    /* ---- tuple plumbing ---- */
    OBM_HD void ensure_line(uint32_t line, uint32_t base) {
        if (line != line_e || base != base_e) {
            if (line >> OBM_LEN_BITS) out.put(OBM_K_LINEHI, line >> OBM_LEN_BITS, 0);
            out.put(OBM_K_LINE, base, line & OBM_MAX_LEN);
            line_e = line; base_e = base;
        }
    }
    OBM_HD void sync_start() { s = p; line_s = line_p; base_s = base_p; }
    /* a slice longer than OBM_MAX_LEN is sent as PART pieces.  Inline on purpose: an out-of-line helper taking the
     * sink by reference would force the sink (and its counters) out of registers into local memory for EVERY put.
     * In the SHORT ASCII instantiations (the hot lexers of the tile and warp kernels) the loop vanishes at compile
     * time; the SHORT Unicode ones keep it here, where it always was, but not in numeric_error. */
    OBM_HD void put_long_prefix(uint32_t &off, uint32_t &len) {
        if (!(ASCII && SHORT)) while (len > OBM_MAX_LEN) { out.put(OBM_K_PART, off, OBM_MAX_LEN); off += OBM_MAX_LEN; len -= OBM_MAX_LEN; }
    }
    /* un-emitted text doc[s,p) becomes a PART (kept in the decoder's pending buffer) */
    OBM_HD void part_tail() {
        if (p > s) {
            ensure_line(line_s, base_s);
            uint32_t off = s, len = p - s;
            put_long_prefix(off, len);
            out.put(OBM_K_PART, off, len);
            sync_start();
        }
    }
    /* emit.go:7-19 */
    OBM_HD void emit(uint32_t kind) {
        ensure_line(line_s, base_s);
        uint32_t off = s, len = p - s;
        put_long_prefix(off, len);
        out.put(kind, off, len);
        last_type = kind;
        sync_start();
    }
    /* emit.go:23-32 */
    OBM_HD void emit_synthetic(uint32_t kind) { out.put(kind, p, 0); last_type = kind; }
    /* discard.go:68-71 */
    OBM_HD void flush() { out.put(OBM_K_FLUSH, p, 0); sync_start(); }
    /* error.go:37-45 (continues in lexComment) / error.go:15-34 (terminates) */
    OBM_HD void located_at_pos(uint32_t kind) { part_tail(); ensure_line(line_p, base_p); out.put(kind, p, 0); }
    /* the literal is quoted in the message and its end p gives the column: a long one goes out as PART pieces and
     * the error tuple keeps off + len = p */
    OBM_HD void numeric_error(uint32_t kind) {
        ensure_line(line_s, base_s);
        uint32_t off = s, len = p - s;
        if (!SHORT) put_long_prefix(off, len);
        out.put(kind, off, len);
    }

    /* ---- reader primitives ---- */
    OBM_HD int peek(uint32_t &w) const {
        if (ASCII) { if (p < n) { w = 1; return (int)d[p]; } w = 0; return RUNE_EOF; }
        return decode_rune(src_raw(d), p, n, w);
    }
    OBM_HD int peek() const { uint32_t w; return peek(w); }
    OBM_HD uint32_t peek_byte() const { return p < n ? d[p] : 0x100u; } /* 0x100 = EOF sentinel */
    /* position.go:18-39 */
    OBM_HD int next() {
        uint32_t w; int r = peek(w);
        last_w = w; last_r = r;
        if (r == RUNE_EOF) return r;
        p += w;
        if (r == '\n') { sv_line = line_p; sv_base = base_p; sv_drift = drift_p; line_p++; base_p = p; drift_p = 0; }
        return r;
    }
    /* position.go:43-57, first call after a next() */
    OBM_HD void backup() {
        if (last_w != 0) {
            p -= last_w;
            if (last_r == '\n') { line_p = sv_line; base_p = sv_base; drift_p = sv_drift; }
        }
    }
    /* position.go:43-57, second call (state.go:79,126): UnreadRune fails, the column still moves */
    OBM_HD void backup_again() {
        if (last_w != 0) { drift_p += last_w; ensure_line(line_p, base_p); out.put(OBM_K_DRIFT, p, 0); }
    }
    /* discard.go:12-38 discard() == discardN(1) */
    OBM_HD void discard1() {
        uint32_t w; int r = peek(w);
        if (r == RUNE_EOF) { flush(); return; }
        part_tail();
        uint32_t adv = (!ASCII && r == RUNE_ERR && w == 1) ? 3u : w; /* utf8.RuneLen(U+FFFD) == 3, discard.go:27-28 */
        if (adv > n - p) adv = n - p;
        p += adv;
        if (r == '\n') { line_p++; base_p = p; drift_p = 0; }
        sync_start();
    }
    /* `q - p` discard() calls over bytes known to be ASCII, non-newline (Accel contract) */
    OBM_HD void discard_to(uint32_t q) {
        if (q > p) { part_tail(); p = q; sync_start(); }
    }
    OBM_HD bool has_prefix2(uint32_t a, uint32_t b) const { return p + 1 < n && d[p] == a && d[p + 1] == b; }
    /* ASCII only.  4-bit mask of the bytes of x that are NOT letters (x's bytes < 0x80):
     * fold case (& 0x5F), then a letter is 0x41..0x5A -- two carry-free byte-wise range adds. */
    static OBM_HD uint32_t nonletter4(uint32_t x) {
        uint32_t y = x & 0x5F5F5F5Fu;
        uint32_t gt = y + 0x25252525u;  /* bit 7 set: y > 0x5A  */
        uint32_t ge = y + 0x3F3F3F3Fu;  /* bit 7 set: y >= 0x41 */
        uint32_t non = (~(ge & ~gt) >> 7) & 0x01010101u;
        return (non * 0x00204081u >> 21) & 0xFu;
    }
    /* Computes the non-letter bits of the 128 bytes starting at the aligned word that holds byte q.  Done
     * once per marker line, by every lane of the warp at the same time (converged): 32 independent word
     * loads and ~10 ALU ops per word.  The window is read as aligned 32-bit words and may extend a few
     * bytes around the document inside the staged buffer; words past the document end are not loaded. */
    OBM_HD void fill_windows(uint32_t q) {
        const uint32_t mis = src_mis(d, q);
        const int32_t w0 = (int32_t)q - (int32_t)mis; /* byte offset of the aligned word that holds byte q */
        const uint32_t wlim = n - q + mis; /* bytes from the window start to the end of the document */
        uint32_t m[4];
#pragma unroll
        for (int g = 0; g < 4; g++) {
            uint32_t mk = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) { const uint32_t wi = (uint32_t)(g * 8 + k); mk |= nonletter4(wi * 4u < wlim ? src_ldw(d, w0 + (int32_t)(wi * 4u)) : 0u) << (4 * k); }
            m[g] = mk;
        }
        wbase = (int32_t)q - (int32_t)mis; wm0 = m[0]; wm1 = m[1]; wm2 = m[2]; wm3 = m[3];
    }
    /* first position >= q (capped at n) whose byte is not an ASCII letter.  Every byte the lexer has to
     * look at (delimiters, quotes, digits, whitespace) is a non-letter, so identifier text is skipped 32
     * bytes per step. */
    OBM_HD uint32_t next_nonletter(uint32_t q) {
        for (;;) {
            if (q >= n) return n;
            const uint32_t sh = (uint32_t)((int32_t)q - wbase);
            if (sh < 128u) {
                const uint32_t g = sh >> 5;
                const uint32_t word = g == 0 ? wm0 : g == 1 ? wm1 : g == 2 ? wm2 : wm3;
                const uint32_t m = word >> (sh & 31u);
                if (m) {
#if defined(__CUDA_ARCH__)
                    q += (uint32_t)(__ffs((int)m) - 1);
#else
                    q += (uint32_t)__builtin_ctz(m);
#endif
                    return q < n ? q : n;
                }
                q = (uint32_t)(wbase + (int32_t)((g + 1u) * 32u));
                continue;
            }
            fill_windows(q); /* beyond the cached 128 bytes (long line): refill from here */
        }
    }

    /* consume.go:65-80 with an ASCII delimiter class; returns `consumed` */
    template <bool NAKED>
    OBM_HD bool consume_until() {
        if (ASCII) { /* '\n' is a delimiter: no line bookkeeping inside the run */
            uint32_t q = p;
            for (;;) {
                q = next_nonletter(q);
                if (q >= n) break;
                uint32_t c = d[q];
                if (NAKED ? is_naked_delim(c) : is_name_delim(c)) break;
                q++; /* digit, '.', '-', '_', '/' ...: part of the name */
            }
            bool any = q > p;
            p = q;
            if (q < n) { last_w = 1; last_r = (int)d[q]; } else { last_w = 0; last_r = RUNE_EOF; } /* state after next()+backup() */
            return any;
        }
        bool consumed = false;
        for (;;) {
            int r = next();
            if (r == RUNE_EOF) { backup(); return consumed; }
            if (r < 0x80 && (NAKED ? is_naked_delim((uint32_t)r) : is_name_delim((uint32_t)r))) { backup(); return consumed; }
            consumed = true;
        }
    }
    OBM_HD bool peeked_whitespaced(const char *tok, uint32_t t, uint32_t &width) const {
        return peeked_whitespaced_at<ASCII>(src_raw(d), n, p, tok, t, width);
    }
    OBM_HD bool peeked_whitespaced_comment(uint32_t &width) const {
        return peeked_whitespaced("//", 2, width) || peeked_whitespaced("#", 1, width);
    }
    /* consume.go:37-47: consumes `width` RUNES (width is a byte count) */
    OBM_HD bool consumed_whitespaced(const char *tok, uint32_t t) {
        uint32_t width;
        if (!peeked_whitespaced(tok, t, width)) return false;
        for (uint32_t k = 0; k < width; k++) next();
        return true;
    }

    /* ---- marker states; each returns the top-level state to continue in ---- */
    /* state.go:60-68, entered with '+' just consumed */
    OBM_HD int marker_start() {
        if (ASCII ? is_letter_ascii(peek()) : is_letter(T, peek())) { emit(OBM_K_MARKER_START); return lex_marker(); }
        return TOP_COMMENT;
    }
    /* ---- ASCII fast machine: the well-formed marker grammar, ONE token (one emit site) per loop
     * iteration so that the lanes of a warp, each lexing its own marker line, stay converged.  It keeps
     * exactly the generic state (p, s, last_type, line basis) and hands over to the generic state
     * functions at a token boundary the moment the input leaves the simple grammar (empty names,
     * missing scope, multi-line / unterminated strings, unusual numbers, leading whitespace, errors),
     * so the tuple stream is the generic one by construction (tests compare them). ---- */
    OBM_HD uint32_t scan_delim(uint32_t q, bool naked) {
        for (;;) {
            q = next_nonletter(q);
            if (q >= n) return n;
            uint32_t c = d[q];
            if (is_name_delim(c) && !(naked && c == ';')) return q;
            q++;
        }
    }
    /* The whole ASCII line machine -- top level (state.go:15-57) and marker grammar -- as ONE loop: every
     * lane of a warp (each lexing its own line) iterates the same loop from the first special byte to the
     * end of its line, so divergence is confined to one iteration (the if-chain rejoins before the single
     * emit site).  Anything outside the simple grammar is handed to the generic state functions at a token
     * boundary; they return the top-level state to continue in. */
    template <bool LINE_MODE>
    OBM_HD int run_ascii() {
        enum { T_LEX, T_COMMENT, F_NAME1, F_COLON, F_ASSIGN, F_VALUE, F_STRBODY, F_STRCLOSE, F_MORE, F_NAME2 };
        enum { X_NONE, X_EOF, X_LINE_END, X_LEX_MARKER, X_LEX_ARGS, X_LEX_VALUE, X_LEX_MORE };
        uint32_t st = T_LEX, send = 0;
        for (;;) {
            uint32_t xc = X_NONE;
            do {
                uint32_t kind = 0, end = p, syn = 0, nst = st;
                bool disc = false;
                if (st <= T_COMMENT) {
                    discard_to(accel.next_interesting(p));
                    end = p;
                    const uint32_t c0 = peek_byte();
                    if (c0 == 0x100u) { if (st == T_LEX) xc = X_EOF; else nst = T_LEX; }
                    else if (c0 == '+') { /* consumed(markerStart) -> lexMarkerStart, state.go:29,48,60-68 */
                        next(); end = p;
                        if (is_letter_ascii((int)peek_byte())) { kind = OBM_K_MARKER_START; nst = F_NAME1; } else nst = T_COMMENT;
                    } else if (st == T_COMMENT) { if (c0 == '\n') nst = T_LEX; else disc = true; }
                    else if (is_space((int)c0)) { disc = true; if (LINE_MODE && c0 == '\n') xc = X_LINE_END; }
                    else if (c0 == '#') { next(); end = p; kind = OBM_K_COMMENT; nst = T_COMMENT; }
                    else if (c0 == '/' && has_prefix2('/', '/')) { next(); next(); end = p; kind = OBM_K_COMMENT; nst = T_COMMENT; }
                    else disc = true;
                } else if (st == F_NAME1 || st == F_NAME2) {
                    end = scan_delim(p, false);
                    const uint32_t c = end < n ? d[end] : 0x100u;
                    const bool term = (c == ' ' || c == '\n' || c == 0x100u);
                    const uint32_t fb = st == F_NAME1 ? X_LEX_MARKER : X_LEX_ARGS;
                    if (end == p) xc = fb;
                    else if (st == F_NAME1 && c == ':') { kind = OBM_K_SCOPE; nst = F_COLON; }
                    else if (st == F_NAME1 && last_type != OBM_K_SEPARATOR) xc = fb;
                    else {
                        kind = OBM_K_ARG;
                        if (c == '=') nst = F_ASSIGN;
                        else if (term) { syn = 3; nst = T_COMMENT; }
                        else if (st == F_NAME2 && c == ',') { syn = 1; nst = F_MORE; }
                        else xc = fb;
                    }
                } else if (st == F_VALUE) {
                    const uint32_t c0 = peek_byte();
                    if (c0 == '\'' || c0 == '"' || c0 == '`') {
                        uint32_t e = p + 1; /* closing quote on this line? */
                        for (;;) { e = next_nonletter(e); if (e >= n) break; uint32_t bb = d[e]; if (bb == c0 || bb == '\n') break; e++; }
                        if (e >= n || d[e] != c0) xc = X_LEX_VALUE;
                        else { send = e; kind = OBM_K_QUOTE; end = p + 1; nst = F_STRBODY; }
                    } else {
                        end = scan_delim(p, true);
                        const uint32_t len = end - p;
                        nst = F_MORE;
                        if (len == 0 || is_space((int)c0)) xc = X_LEX_VALUE; /* \t \v \f \r may lead a bool literal (consume.go:37-47) */
                        else if (c0 == '.' || c0 == '-' || is_digit_ascii((int)c0)) {
                            /* -?digits[.digits], at most 17 bytes: valid and in range for Atoi / ParseFloat */
                            uint32_t dots = 0, digits = 0; bool ok = len <= 17;
                            for (uint32_t k = (c0 == '-') ? 1u : 0u; ok && k < len; k++) {
                                uint32_t bb = d[p + k];
                                if (bb == '.') dots++; else if (bb >= '0' && bb <= '9') digits++; else ok = false;
                            }
                            if (!ok || dots > 1 || digits == 0) xc = X_LEX_VALUE;
                            kind = dots ? OBM_K_FLOAT_LITERAL : OBM_K_INTEGER_LITERAL;
                        } else {
                            const bool t4 = len >= 4 && d[p] == 't' && d[p + 1] == 'r' && d[p + 2] == 'u' && d[p + 3] == 'e';
                            const bool f5 = len >= 5 && d[p] == 'f' && d[p + 1] == 'a' && d[p + 2] == 'l' && d[p + 3] == 's' && d[p + 4] == 'e';
                            if ((t4 && len > 4) || (f5 && len > 5)) xc = X_LEX_VALUE;
                            kind = (t4 || f5) ? OBM_K_BOOL_LITERAL : OBM_K_STRING_LITERAL;
                        }
                    }
                } else if (st == F_MORE) {
                    const uint32_t c0 = peek_byte();
                    if (c0 == ',') { kind = OBM_K_ARG_DELIMITER; end = p + 1; nst = F_NAME2; }
                    else if (c0 == ' ' || c0 == '\n' || c0 == 0x100u) { syn = 2; nst = T_COMMENT; }
                    else xc = X_LEX_MORE;
                } else if (st == F_STRBODY) { kind = OBM_K_STRING_LITERAL; end = send; nst = F_STRCLOSE; }
                else { /* single-byte tokens: ':' '=' closing quote */
                    kind = st == F_COLON ? OBM_K_SEPARATOR : st == F_ASSIGN ? OBM_K_ARG_ASSIGNMENT : OBM_K_QUOTE;
                    end = p + 1;
                    nst = st == F_COLON ? F_NAME1 : st == F_ASSIGN ? F_VALUE : F_MORE;
                }
                if (xc == X_NONE || xc == X_LINE_END) {
                    if (disc) discard1();
                    if (kind) { p = end; emit(kind); }
                    if (syn & 1u) emit_synthetic(OBM_K_SYNTHETIC_BOOL);
                    if (syn & 2u) emit_synthetic(OBM_K_MARKER_END);
                    st = nst;
                }
                OBM_OPAQUE(st);
                OBM_OPAQUE(xc);
            } while (xc == X_NONE);
            if (xc == X_EOF) { if (!LINE_MODE) out.put(OBM_K_EOF, n, 0); return RUN_EOF; }
            if (xc == X_LINE_END) return RUN_LINE_END;
            /* one hand-over point per generic entry */
            int top = xc == X_LEX_MARKER ? lex_marker() : xc == X_LEX_VALUE ? lex_arg_value() : lex_more_args(xc == X_LEX_ARGS);
            if (top == TOP_FATAL) return RUN_FATAL;
            st = top == TOP_LEX ? T_LEX : T_COMMENT;
        }
    }

    /* state.go:71-116 */
    OBM_HD int lex_marker() {
        for (;;) {
            if (!consume_until<false>()) { backup_again(); flush(); return TOP_COMMENT; }
            uint32_t c = peek_byte();
            if (c == ':') { emit(OBM_K_SCOPE); next(); emit(OBM_K_SEPARATOR); continue; }
            if (c == ' ' || c == '\n' || c == 0x100u) {
                if (last_type != OBM_K_SEPARATOR) { located_at_pos(OBM_K_WARN_NOSCOPE); return TOP_COMMENT; }
                emit(OBM_K_ARG); emit_synthetic(OBM_K_SYNTHETIC_BOOL); emit_synthetic(OBM_K_MARKER_END);
                return TOP_COMMENT;
            }
            if (c == '=') {
                if (last_type != OBM_K_SEPARATOR) { located_at_pos(OBM_K_WARN_NOSCOPE); return TOP_COMMENT; }
                emit(OBM_K_ARG); next(); emit(OBM_K_ARG_ASSIGNMENT);
                return lex_arg_value();
            }
            located_at_pos(OBM_K_WARN_INVALID);
            return TOP_COMMENT;
        }
    }
    /* state.go:118-154 (lexArgs) and state.go:304-317 (lexMoreArgs), as one loop */
    OBM_HD int lex_more_args(bool at_args = false) {
        for (;;) {
            uint32_t c;
            if (!at_args) {
                c = peek_byte();
                if (c == ',') { next(); emit(OBM_K_ARG_DELIMITER); }
                else if (c == ' ' || c == '\n' || c == 0x100u) { emit_synthetic(OBM_K_MARKER_END); return TOP_COMMENT; }
                else { located_at_pos(OBM_K_ERR_MALFORMED); return TOP_FATAL; }
            }
            at_args = false;
            /* lexArgs */
            if (!consume_until<false>()) { backup_again(); flush(); emit_synthetic(OBM_K_MARKER_END); return TOP_LEX; }
            emit(OBM_K_ARG);
            c = peek_byte();
            if (c == '=') { next(); emit(OBM_K_ARG_ASSIGNMENT); int st = lex_arg_value_inner(); if (st != -1) return st; continue; }
            if (c == ' ' || c == '\n' || c == 0x100u) { emit_synthetic(OBM_K_SYNTHETIC_BOOL); emit_synthetic(OBM_K_MARKER_END); return TOP_COMMENT; }
            if (c == ',') { emit_synthetic(OBM_K_SYNTHETIC_BOOL); continue; }
            located_at_pos(OBM_K_ERR_MALFORMED);
            return TOP_FATAL;
        }
    }
    OBM_HD int lex_arg_value() { int st = lex_arg_value_inner(); return st != -1 ? st : lex_more_args(); }
    /* state.go:156-302; returns -1 to continue in lexMoreArgs, else a TopState (fatal) */
    OBM_HD int lex_arg_value_inner() {
        uint32_t c = peek_byte();
        /* lexStringLiteral, state.go:176-221 */
        if (c == '\'' || c == '"' || c == '`') {
            next(); emit(OBM_K_QUOTE);
            for (;;) {
                if (ASCII) p = next_nonletter(p); /* quotes and newlines are non-letters */
                uint32_t b = peek_byte();
                if (b == 0x100u) { located_at_pos(OBM_K_ERR_UNMATCHED); return TOP_FATAL; }
                if (b == '\n') {
                    if (c != '`') { located_at_pos(OBM_K_ERR_UNMATCHED); return TOP_FATAL; }
                    next();
                    uint32_t width;
                    if (peeked_whitespaced_comment(width)) {
                        while (!(has_prefix2('/', '/') || peek_byte() == '#')) discard1(); /* discardUntil */
                        discard1();
                    }
                } else if (b == c) {
                    emit(OBM_K_STRING_LITERAL); next(); emit(OBM_K_QUOTE);
                    return -1;
                } else {
                    next();
                }
            }
        }
        /* lexNumericLiteral, state.go:223-276 */
        {
            int r0 = peek();
            if (r0 == '.' || r0 == '-' || (ASCII ? is_digit_ascii(r0) : is_number(T, r0))) {
                bool isfloat = (r0 == '.');
                for (;;) {
                    next();
                    uint32_t b = peek_byte();
                    if (b == '.' || b == 'e' || b == 'E' || b == '-') { isfloat = true; continue; }
                    if (!(ASCII ? is_digit_ascii(peek()) : is_number(T, peek()))) break;
                }
                int code = isfloat ? parse_float_err(T, src_raw(d) + s, p - s) : atoi_err(src_raw(d) + s, p - s);
                if (code) { numeric_error(isfloat ? OBM_K_ERR_FLOAT : OBM_K_ERR_INT); return TOP_FATAL; }
                emit(isfloat ? OBM_K_FLOAT_LITERAL : OBM_K_INTEGER_LITERAL);
                return -1;
            }
        }
        /* lexBooleanLiteral, state.go:278-286 */
        if (consumed_whitespaced("true", 4) || consumed_whitespaced("false", 5)) { emit(OBM_K_BOOL_LITERAL); return -1; }
        /* lexNakedStringLiteral, state.go:288-302 */
        if (consume_until<true>()) { emit(OBM_K_STRING_LITERAL); return -1; }
        located_at_pos(OBM_K_ERR_MALFORMED);
        return TOP_FATAL;
    }

    /* ---- top level: state.go:15-57.  LINE_MODE (the tile path's per-line owner) stops right after
     *      discarding the first top-level '\n'; otherwise runs to EOF and emits the EOF tuple. ---- */
    template <bool LINE_MODE>
    OBM_HD int run() {
        if (ASCII) return run_ascii<LINE_MODE>();
        int st = TOP_LEX;
        for (;;) {
            if (st == TOP_LEX) {
                discard_to(accel.next_interesting(p));
                uint32_t w; int r = peek(w);
                if (r == RUNE_EOF) { if (!LINE_MODE) out.put(OBM_K_EOF, n, 0); return RUN_EOF; }
                if (is_space(r)) {
                    discard1();
                    if (LINE_MODE && r == '\n') return RUN_LINE_END;
                    continue;
                }
                if (has_prefix2('/', '/')) { next(); next(); emit(OBM_K_COMMENT); st = TOP_COMMENT; }
                else if (r == '#') { next(); emit(OBM_K_COMMENT); st = TOP_COMMENT; }
                else if (r == '+') { next(); st = marker_start(); }
                else discard1();
            } else if (st == TOP_COMMENT) {
                discard_to(accel.next_interesting(p));
                uint32_t c = peek_byte();
                if (c == '+') { next(); st = marker_start(); }
                else if (c == '\n' || c == 0x100u) st = TOP_LEX;
                else discard1();
            } else {
                return RUN_FATAL;
            }
        }
    }
};

} /* namespace obm */
#endif /* OBM_CORE_H */
