/*
 * obm_warp.h -- host/device logic of the fused, warp-autonomous scan (mode 0 since round 2).
 *
 * One WARP owns a unit: the documents that start inside a TILE-byte range of the packed batch (at most DMAX of
 * them, at most BUFB bytes).  The unit's text is staged once into the warp's slice of shared memory (TMA bulk
 * copy, obm_warp.cuh) and everything else happens inside the warp, without a block barrier and without a
 * second read of the text from HBM:
 *
 *   A  steps     2 KiB per step, 64 contiguous bytes per lane: SIMD-within-register byte classes -> newline / special
 *                bitmaps ('#', '+', "//": what can start a comment or a marker in lex / lexComment,
 *                state.go:20-33,48), bit-parallel "first special of every line" ((~events + starts) & events with
 *                a ballot carry look-ahead across lanes), newline prefix counts -> owner list in position order
 *   B  owners    a lane per owning line: line start, line number, document; plain comment line or marker line
 *   C  markers   marker lines compacted, a lane per line: the branch-light stepper below (fast_line) walks the
 *                well-formed grammar  +scope:scope:arg=value,arg=value  token by token from the shared-memory
 *                text and stages packed 4-byte tuples; anything else is handed to the generic obm::Lexer
 *                (obm_core.h) -- the same hand-over rule as r01's run_ascii, so there is one source of truth
 *   D  assemble  tuple counts -> warp scans -> unit total -> two-level decoupled look-back over units -> final
 *                positions; plain / EOF tuples are written in place, staged marker tuples lane-per-tuple
 *
 * Documents the line-parallel view cannot represent (bytes >= 0x80, lines that interact across a newline, a
 * fatal error, more owners than OWN_CAP) are lexed sequentially by the exact Unicode lexer inside the same warp,
 * exactly as in r01 (obmp::doc_exact).  The tuple stream is the canonical one (DESIGN.md section 3).
 *
 * Everything in this header compiles for the host too: tests/hostsim replays a warp with 32 fibers
 * (tests/hostsim/warp_emu.h) and compares with the exact path and the oracle.
 */
#ifndef OBM_WARP_H
#define OBM_WARP_H

#include "obm_pipe.h"

#ifndef OBMW_TILE
#define OBMW_TILE 12288
#endif
#ifndef OBMW_BUFB
#define OBMW_BUFB 13312
#endif

namespace obmw {

constexpr uint32_t TILE = OBMW_TILE;      /* a unit = the documents starting in [t*TILE, (t+1)*TILE) (split when > DMAX / > BUFB) */
constexpr uint32_t BUFB = OBMW_BUFB;      /* bytes of text staged per warp */
constexpr uint32_t MAXDOC = (BUFB - 16 < 16368u) ? BUFB - 16 : 16368u; /* larger documents take the chunk-parallel exact path */
constexpr uint32_t ROW = 1024;            /* bytes per bitmap row: 32 words, one W.naw entry */
constexpr uint32_t STEP = 2048;           /* bytes per phase-A step: 64 per lane, words 2L and 2L+1 (one W.nlpre entry) */
constexpr uint32_t NWORDS = BUFB / 32;    /* 32-byte words of the bitmaps */
constexpr uint32_t DMAX = 31;             /* documents per unit: one lane each, lane nd holds the end */
constexpr uint32_t OWN_CAP = 256;         /* owning lines per unit (more: the unit is paged, document by document; a document with more: the exact lexer) */
constexpr uint32_t MLCAP = 32;            /* marker lines whose tuples are staged: one per lane */
constexpr uint32_t LTS = 24;              /* staged tuples per marker line */
constexpr uint32_t FIN_CAP = TILE / 16 - 64; /* tuples of a unit whose write is deferred (0.46 B of tuples per input byte: manifests need 0.35) */
static_assert(BUFB % ROW == 0 && BUFB >= TILE + 16 && BUFB <= 16384 + ROW, "buffer geometry");

/* document flags; DF_UNI lives only between phases A and B: a valid-UTF-8 document without Unicode white space stays on the
 * line-parallel path unless one of its MARKER lines holds bytes >= 0x80 (then: the exact lexer, DF_INTERACT) */
enum : uint32_t { DF_NONASCII = 1, DF_INTERACT = 2, DF_QOVERFLOW = 4, DF_UNI = 8, DF_EXACT = 7 };
enum : uint32_t { PD_GENERIC = 255 /* orec plusd: the line is the generic ASCII lexer's */ };

/* ---- owner record (8 bytes), positions document-relative ------------------------------------------------
 *  0..13 ls | 14..27 first special | 28..41 line | 42 marker | 43 slash2 ("//" comment) | 44 dead (no tuple)
 *  45..49 document (index inside the unit) | 50..57 plus - first (marker lines; 255: not known) */
typedef uint64_t orec_t;
OBM_HD orec_t make_orec(uint32_t ls, uint32_t first, uint32_t line, bool marker, bool slash2, bool dead, uint32_t d, uint32_t plusd) {
    return (orec_t)ls | ((orec_t)first << 14) | ((orec_t)line << 28) | ((orec_t)marker << 42) | ((orec_t)slash2 << 43) |
           ((orec_t)dead << 44) | ((orec_t)d << 45) | ((orec_t)plusd << 50);
}
OBM_HD uint32_t or_ls(orec_t r) { return (uint32_t)(r & 0x3FFF); }
OBM_HD uint32_t or_first(orec_t r) { return (uint32_t)((r >> 14) & 0x3FFF); }
OBM_HD uint32_t or_line(orec_t r) { return (uint32_t)((r >> 28) & 0x3FFF); }
OBM_HD bool or_marker(orec_t r) { return (r >> 42) & 1; }
OBM_HD bool or_slash2(orec_t r) { return (r >> 43) & 1; }
OBM_HD bool or_dead(orec_t r) { return (r >> 44) & 1; }
OBM_HD uint32_t or_doc(orec_t r) { return (uint32_t)((r >> 45) & 0x1F); }
OBM_HD uint32_t or_plusd(orec_t r) { return (uint32_t)((r >> 50) & 0xFF); }

/* ---- staged tuple (4 bytes): kind 5 | len 13 | off 14 (document-relative) -------------------------------- */
constexpr uint32_t ST_MAXOFF = (1u << 14) - 1u, ST_MAXLEN = (1u << 13) - 1u;
OBM_HD uint32_t st_pack(uint32_t kind, uint32_t off, uint32_t len) { return (kind << 27) | (len << 14) | off; }
OBM_HD obm_tuple st_unpack(uint32_t v) { /* kind stays in the top 5 bits of the high word */
    return ((uint64_t)((v & 0xF8000000u) | ((v >> 14) & ST_MAXLEN)) << 32) | (uint64_t)(v & ST_MAXOFF);
}

/* sink of the stepper: packed into the warp's staging slot (cap LTS), counts always */
struct PackSink {
    uint32_t *st; uint32_t cap, n, mk, lx; bool ovf;
    OBM_HD PackSink(uint32_t *s, uint32_t c) : st(s), cap(c), n(0), mk(0), lx(0), ovf(false) {}
    OBM_HD void put(uint32_t kind, uint32_t off, uint32_t len) {
        if (n < cap && len <= ST_MAXLEN) st[n] = st_pack(kind, off, len); else ovf = true;
        n++;
        mk += (kind == OBM_K_MARKER_START);
        lx += (kind - (uint32_t)OBM_K_PART) > 4u;
    }
};
/* sink of the stepper: straight to the final place in global memory */
struct DirectSink {
    obm_tuple *out; uint32_t cap, n, mk, lx; bool ovf;
    OBM_HD DirectSink(obm_tuple *o, uint32_t c) : out(o), cap(c), n(0), mk(0), lx(0), ovf(false) {}
    OBM_HD void put(uint32_t kind, uint32_t off, uint32_t len) {
        if (n < cap) out[n] = OBM_TUPLE(kind, off, len);
        n++;
        mk += (kind == OBM_K_MARKER_START);
        lx += (kind - (uint32_t)OBM_K_PART) > 4u;
    }
};

#if defined(__CUDA_ARCH__)
#define OBMW_FFS(x) ((uint32_t)__ffs((int)(x)))
#define OBMW_FFS64(x) ((uint32_t)__ffsll((long long)(x)))
#define OBMW_POPC64(x) ((uint32_t)__popcll(x))
#define OBMW_FUNNEL_L(lo, hi, s) __funnelshift_l((lo), (hi), (s))
#else
#define OBMW_FFS(x) ((uint32_t)__builtin_ffs((int)(x)))
#define OBMW_FFS64(x) ((uint32_t)__builtin_ffsll((long long)(x)))
#define OBMW_POPC64(x) ((uint32_t)__builtin_popcountll(x))
#define OBMW_FUNNEL_L(lo, hi, s) ((uint32_t)(((((uint64_t)(hi)) << 32) | (uint64_t)(lo)) << ((s) & 31) >> 32))
#endif

/* ---- A: byte classes of 32 bytes (8 little-endian words) ------------------------------------------------ */
struct Masks { uint32_t nl, hp, sl, hi; };
/* bit 7 of every byte of the result: the byte of t is zero.  7-bit form: t's bytes must be < 0x80. */
OBM_HD uint32_t zflag7(uint32_t t) { return ~(t + 0x7F7F7F7Fu) & 0x80808080u; }
OBM_HD uint32_t zflag8(uint32_t t) { return ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t) & 0x80808080u; }
/* flags at bits 7,15,23,31 -> 4 bits appended below acc's (acc holds the masks of the HIGHER words) */
OBM_HD uint32_t nib_append(uint32_t acc, uint32_t z) { return OBMW_FUNNEL_L(z * 0x00204081u, acc, 4); }
template <bool EXACT>
OBM_HD Masks classify32_t(const uint32_t (&x)[8]) {
    Masks m{0, 0, 0, 0};
#pragma unroll
    for (int k = 7; k >= 0; k--) {
        const uint32_t v = x[k];
        m.hi |= v;
        const uint32_t tn = v ^ 0x0A0A0A0Au, th = (v & 0xF7F7F7F7u) ^ 0x23232323u /* '#' 0x23 or '+' 0x2B */, ts = v ^ 0x2F2F2F2Fu;
        m.nl = nib_append(m.nl, EXACT ? zflag8(tn) : zflag7(tn));
        m.hp = nib_append(m.hp, EXACT ? zflag8(th) : zflag7(th));
        m.sl = nib_append(m.sl, EXACT ? zflag8(ts) : zflag7(ts));
    }
    m.hi &= 0x80808080u;
    return m;
}
OBM_HD Masks classify32(const uint32_t (&x)[8]) {
    Masks m = classify32_t<false>(x);
    if (m.hi) { const uint32_t hi = m.hi; m = classify32_t<true>(x); m.hi = hi; } /* bytes >= 0x80: the carry-free test is only exact for 7-bit input */
    return m;
}
/* bits of [pos0, pos0+32) that lie inside [lo, hi) */
OBM_HD uint32_t range_mask(uint32_t pos0, uint32_t lo, uint32_t hi) {
    uint32_t keep = 0xFFFFFFFFu;
    if (lo > pos0) keep &= (lo - pos0 >= 32u) ? 0u : (0xFFFFFFFFu << (lo - pos0));
    if (hi < pos0 + 32u) keep &= (hi <= pos0) ? 0u : (0xFFFFFFFFu >> (pos0 + 32u - hi));
    return keep;
}
/* bits of [pos0, pos0+64) that lie inside [lo, hi) */
OBM_HD uint64_t range_mask64(uint32_t pos0, uint32_t lo, uint32_t hi) {
    uint64_t keep = ~0ull;
    if (lo > pos0) keep &= (lo - pos0 >= 64u) ? 0ull : (~0ull << (lo - pos0));
    if (hi < pos0 + 64u) keep &= (hi <= pos0) ? 0ull : (~0ull >> (pos0 + 64u - hi));
    return keep;
}
/* bits 0..15 of v to the even bits 0, 2, .., 30 */
OBM_HD uint32_t spread16(uint32_t v) {
    v &= 0xFFFFu;
    v = (v | (v << 8)) & 0x00FF00FFu; v = (v | (v << 4)) & 0x0F0F0F0Fu;
    v = (v | (v << 2)) & 0x33333333u; v = (v | (v << 1)) & 0x55555555u;
    return v;
}

/* ---- C: the stepper ------------------------------------------------------------------------------------
 * Text access: Src is a byte source indexed by buffer-relative position (obm_core.h: const uint8_t* or ShBytes);
 * the buffer base is 16-byte aligned, so position & 3 is the alignment of an aligned-word load. */
template <class Src> OBM_HD uint32_t tw_ldw(const Src &t, uint32_t pos_aligned) { return obm::src_ldw(t, (int32_t)pos_aligned); }

/* bit 7 of each byte: the byte is NOT one of [0-9A-Za-z] '-' '.' '/' (nor 0x0D..0x19): a superset of the name
 * delimiters (state.go:72-76), exact for 7-bit bytes.  Case fold (& 0x5F) maps letters to 0x41..0x5A and
 * 0x2D..0x39 to 0x0D..0x19; two carry-free range tests per class. */
OBM_HD uint32_t nonname4(uint32_t w) {
    const uint32_t y = w & 0x5F5F5F5Fu;
    const uint32_t letter = (y + 0x3F3F3F3Fu) & ~(y + 0x25252525u);   /* 0x41 <= y <= 0x5A */
    const uint32_t digit = (y + 0x73737373u) & ~(y + 0x66666666u);    /* 0x0D <= y <= 0x19 */
    return ~(letter | digit) & 0x80808080u;
}
/* 16 flag bytes (bit 7 of each byte of z[0..3]) -> 16-bit mask, bit i = byte i */
OBM_HD uint32_t flags16(const uint32_t (&z)[4]) {
    uint32_t m = 0;
#pragma unroll
    for (int k = 3; k >= 0; k--) m = nib_append(m, z[k]);
    return m;
}
/* first position q in [p, lim) whose byte is a name delimiter (naked: ';' does not count), else lim.  16 bytes per step
 * (one 128-bit shared-memory load, four independent class computations): the lexer is latency-bound, not issue-bound */
template <class Src>
OBM_HD uint32_t scan_delim(const Src &t, uint32_t p, uint32_t lim, bool naked) {
    uint32_t a = p & ~15u;
    uint32_t from = 0xFFFFu << (p & 15u);
    for (;;) {
        const obm::Quad q4 = obm::src_ldq(t, a);
        const uint32_t z[4] = {nonname4(q4.w[0]), nonname4(q4.w[1]), nonname4(q4.w[2]), nonname4(q4.w[3])};
        uint32_t m = flags16(z) & from;
        while (m) {
            const uint32_t q = a + OBMW_FFS(m) - 1u;
            if (q >= lim) return lim;
            const uint32_t c = t[q];
            if (obm::is_name_delim(c) && !(naked && c == ';')) return q;
            m &= m - 1u;
        }
        a += 16u; from = 0xFFFFu;
        if (a >= lim) return lim;
    }
}
/* first position q in [p, lim) whose byte equals c (7-bit) or '\n', else lim */
template <class Src>
OBM_HD uint32_t scan_byte_or_nl(const Src &t, uint32_t p, uint32_t lim, uint32_t c) {
    const uint32_t rep = c * 0x01010101u;
    uint32_t a = p & ~15u;
    uint32_t from = 0xFFFFu << (p & 15u);
    for (;;) {
        const obm::Quad q4 = obm::src_ldq(t, a);
        uint32_t z[4];
#pragma unroll
        for (int k = 0; k < 4; k++) z[k] = zflag8(q4.w[k] ^ rep) | zflag8(q4.w[k] ^ 0x0A0A0A0Au); /* exact form: the 16 bytes may hold a neighbour's bytes >= 0x80 */
        const uint32_t m = flags16(z) & from;
        if (m) { const uint32_t q = a + OBMW_FFS(m) - 1u; return q < lim ? q : lim; }
        a += 16u; from = 0xFFFFu;
        if (a >= lim) return lim;
    }
}

enum : uint32_t { FL_OK = 0, FL_FALLBACK = 1 };

/* One marker line of an all-ASCII document, from the shared-memory text.  first: the line's first special byte
 * ('#', "//" or '+'); plus: the first '+' at or after it; ls / line: start and number of the line; [dpos, dend):
 * the document.  All positions buffer-relative; tuples carry document-relative offsets.  Emits exactly what
 * obm::Lexer<.., ASCII> in LINE mode emits for the line (state.go:15-317) as long as the line stays inside the
 * well-formed grammar; returns FL_FALLBACK (sink contents void) the moment it does not:
 *   '+' not followed by a letter (stale buffer, A.4b), empty names (column drift, A.6), a marker without scope or
 *   an invalid one (warnings), strings that do not close on the line, numbers other than -?digits[.digits] of at
 *   most 17 bytes, leading white space / longer words after true|false, malformed arguments (fatal). */
template <class Src, class Sink>
OBM_HD uint32_t fast_line(const Src &t, uint32_t first, uint32_t plus, uint32_t ls, uint32_t line, uint32_t dpos, uint32_t dend, Sink &o) {
    if (!(line == 1 && ls == dpos)) o.put(OBM_K_LINE, ls - dpos, line);
    {
        const uint32_t c = t[first];
        if (c == '#') o.put(OBM_K_COMMENT, first - dpos, 1);
        else if (c == '/') o.put(OBM_K_COMMENT, first - dpos, 2);
    }
    uint32_t p = plus;
    for (;;) { /* one marker per iteration; p at its '+' */
        if (!(p + 1 < dend && obm::is_letter_ascii((int)t[p + 1]))) return FL_FALLBACK;
        o.put(OBM_K_MARKER_START, p - dpos, 1);
        p++;
        uint32_t e, c, nscopes = 0;
        for (;;) { /* lexMarker, state.go:71-116 */
            e = scan_delim(t, p, dend, false);
            c = e < dend ? (uint32_t)t[e] : 0x100u;
            if (e == p) return FL_FALLBACK;
            if (c != ':') break;
            o.put(OBM_K_SCOPE, p - dpos, e - p);
            o.put(OBM_K_SEPARATOR, e - dpos, 1);
            p = e + 1; nscopes++;
        }
        if (nscopes == 0) return FL_FALLBACK;
        if (!(c == '=' || c == ' ' || c == '\n' || c == 0x100u)) return FL_FALLBACK; /* first argument: "invalid marker" otherwise */
        for (;;) { /* one argument per iteration: name [p, e), c = the byte behind it */
            o.put(OBM_K_ARG, p - dpos, e - p);
            p = e;
            if (c == '=') {
                o.put(OBM_K_ARG_ASSIGNMENT, p - dpos, 1);
                p++;
                const uint32_t c0 = p < dend ? (uint32_t)t[p] : 0x100u;
                if (c0 == '\'' || c0 == '"' || c0 == '`') { /* lexStringLiteral, state.go:176-221, closing on this line */
                    const uint32_t q = scan_byte_or_nl(t, p + 1, dend, c0);
                    if (q >= dend || (uint32_t)t[q] != c0) return FL_FALLBACK;
                    o.put(OBM_K_QUOTE, p - dpos, 1);
                    o.put(OBM_K_STRING_LITERAL, p + 1 - dpos, q - p - 1);
                    o.put(OBM_K_QUOTE, q - dpos, 1);
                    p = q + 1;
                } else {
                    const uint32_t e2 = scan_delim(t, p, dend, true);
                    const uint32_t len = e2 - p;
                    if (len == 0 || obm::is_space((int)c0)) return FL_FALLBACK;
                    uint32_t kind;
                    if (c0 == '.' || c0 == '-' || obm::is_digit_ascii((int)c0)) { /* state.go:223-276 for -?digits[.digits] */
                        uint32_t dots = 0, digits = 0; bool ok = len <= 17;
                        for (uint32_t k = (c0 == '-') ? 1u : 0u; ok && k < len; k++) {
                            const uint32_t bb = t[p + k];
                            if (bb == '.') dots++; else if (bb >= '0' && bb <= '9') digits++; else ok = false;
                        }
                        if (!ok || dots > 1 || digits == 0) return FL_FALLBACK;
                        kind = dots ? OBM_K_FLOAT_LITERAL : OBM_K_INTEGER_LITERAL;
                    } else {
                        kind = OBM_K_STRING_LITERAL;
                        if (c0 == 't' || c0 == 'f') { /* true / false; a longer word that starts with one of them is the generic lexer's (A.7) */
                            const bool t4 = len >= 4 && c0 == 't' && t[p + 1] == 'r' && t[p + 2] == 'u' && t[p + 3] == 'e';
                            const bool f5 = len >= 5 && c0 == 'f' && t[p + 1] == 'a' && t[p + 2] == 'l' && t[p + 3] == 's' && t[p + 4] == 'e';
                            if ((t4 && len > 4) || (f5 && len > 5)) return FL_FALLBACK;
                            if (t4 || f5) kind = OBM_K_BOOL_LITERAL;
                        }
                    }
                    o.put(kind, p - dpos, len);
                    p = e2;
                }
                c = p < dend ? (uint32_t)t[p] : 0x100u; /* lexMoreArgs, state.go:304-317 */
                if (c == ' ' || c == '\n' || c == 0x100u) { o.put(OBM_K_MARKER_END, p - dpos, 0); break; }
                if (c != ',') return FL_FALLBACK;
            } else if (c == ',') { /* a flag followed by another argument (lexArgs, state.go:140-141) */
                o.put(OBM_K_SYNTHETIC_BOOL, p - dpos, 0);
            } else { /* ' ', '\n', end: a flag closes the marker */
                o.put(OBM_K_SYNTHETIC_BOOL, p - dpos, 0);
                o.put(OBM_K_MARKER_END, p - dpos, 0);
                break;
            }
            /* p at ',' */
            o.put(OBM_K_ARG_DELIMITER, p - dpos, 1);
            p++;
            e = scan_delim(t, p, dend, false);
            if (e == p) return FL_FALLBACK;
            c = e < dend ? (uint32_t)t[e] : 0x100u;
            if (!(c == '=' || c == ',' || c == ' ' || c == '\n' || c == 0x100u)) return FL_FALLBACK;
        }
        /* lexComment (state.go:46-57): the next '+' on this line starts another marker */
        const uint32_t q = scan_byte_or_nl(t, p, dend, '+');
        if (q >= dend || (uint32_t)t[q] != '+') return FL_OK;
        p = q;
    }
}

/* ---- units: tile -> (first document, last document, flags), computed by k_wunits / the host replay -------- */
struct WRec { uint32_t d_first; uint32_t d_last; uint32_t flags; uint32_t n_units; };
enum : uint32_t { WR_LARGE = 1 /* the tile's last document takes the large path */, WR_SPLIT = 2 /* ... gets a unit of its own */ };
/* units of tile [d0, d1): groups of <= DMAX small documents that fit the buffer; the last document is set apart when
 * it is large (chunk-parallel exact path) or when it would not fit together with the others */
OBM_HD WRec make_wrec(const uint64_t *doc_off, uint32_t d0, uint32_t d1) {
    WRec r{d0, d1, 0, 0};
    if (d1 == d0) return r;
    const uint32_t large = (doc_off[d1] - doc_off[d1 - 1] > MAXDOC) ? 1u : 0u;
    const uint32_t ns = d1 - d0 - large;
    if (large) r.flags |= WR_LARGE;
    if (ns == 0) { r.n_units = 1; return r; }
    const uint64_t span = doc_off[d0 + ns] - doc_off[d0];
    if (span + 15u <= BUFB || ns == 1) r.n_units = (ns + DMAX - 1) / DMAX;
    else { r.flags |= WR_SPLIT; r.n_units = (ns - 1 + DMAX - 1) / DMAX + 1; }
    return r;
}
/* unit k of the tile: documents [da, db) (possibly none), extra = the tile's large document closes this unit */
OBM_HD void wrec_unit(const WRec &r, uint32_t k, uint32_t &da, uint32_t &db, uint32_t &extra) {
    const uint32_t large = (r.flags & WR_LARGE) ? 1u : 0u;
    const uint32_t small_end = r.d_last - large;
    const uint32_t group_end = (r.flags & WR_SPLIT) ? small_end - 1 : small_end;
    da = r.d_first + k * DMAX;
    if (da >= group_end && (r.flags & WR_SPLIT) && k == r.n_units - 1) { da = group_end; db = small_end; }
    else { db = da + DMAX < group_end ? da + DMAX : group_end; if (da > db) da = db; }
    extra = (large && k == r.n_units - 1) ? 1u : 0u;
}

} /* namespace obmw */
#endif
