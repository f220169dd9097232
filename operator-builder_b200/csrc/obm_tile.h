/*
 * obm_tile.h -- the tile fast path's per-thread phase logic, written as host/device functions over
 * a shared-memory image (`obmt::Smem`) so that tests/hostsim can replay a CTA phase by phase on the
 * CPU.  The CUDA kernel (obm_fast.cuh) supplies the data movement (TMA bulk copy into Smem::data),
 * the barriers between phases, the warp-shuffle scans and the cross-CTA look-back.
 *
 * One CTA owns the documents that START inside a TILE-byte range of the packed batch.  Documents of
 * at most MAXDOC bytes are staged whole in shared memory and lexed line-parallel:
 *
 *   P2 classify     every 32-byte word -> newline bitmap, special bitmap ('#', '+', "//": everything that
 *                   can start a comment or a marker), non-ASCII flag
 *   P3 doc prep     a virtual newline in front of every document start; per-document non-ASCII flag
 *   P4 line scan    newline prefix counts (line numbers) + "owners": looking forward from every
 *                   (virtual) newline, a line that contains a '+' becomes a MARKER owner, a line with
 *                   only a comment start becomes a PLAIN owner, any other line produces no tuple
 *                   (reference semantics: a line starts in state `lex`, SURVEY.md A.11)
 *   P5 owners       plain owners: 1-2 tuples, computed in place.  Marker owners are compacted into a
 *                   dense list; one thread per marker line runs the ASCII instantiation of obm::Lexer
 *                   in LINE mode from the line's first special byte and stages its tuples in shared
 *                   memory
 *   P6 resolve      documents whose lines interact (multi-line literal, fatal error) or that contain
 *                   non-ASCII bytes are re-lexed sequentially by one thread (exact path, same core);
 *                   tuple counts -> offsets
 *   P7 fill         staged tuples are copied to their final global positions (a warp per owner)
 *
 * The tuple stream is identical to the exact path's by construction (same obm::Lexer, canonical
 * LINE/PART rules); tests compare the two streams tuple for tuple.
 */
#ifndef OBM_TILE_H
#define OBM_TILE_H

#include <stdint.h>
#include "obm_core.h"

#if defined(__CUDA_ARCH__)
#define OBMT_POPC(x) ((uint32_t)__popc(x))
#define OBMT_CTZ(x) ((uint32_t)(__ffs((int)(x)) - 1))
#else
#define OBMT_POPC(x) ((uint32_t)__builtin_popcount(x))
#define OBMT_CTZ(x) ((uint32_t)__builtin_ctz(x))
#endif

namespace obmt {

constexpr uint32_t NT = 256;        /* threads per CTA */
constexpr uint32_t TILE = 16384;    /* a CTA owns the documents starting in [t*TILE, (t+1)*TILE) */
constexpr uint32_t MAXDOC = 16368;  /* documents up to this size take the tile path */
constexpr uint32_t NW = 1024;       /* 32-byte words staged per sub-batch (32 KiB) */
constexpr uint32_t WPT = NW / NT;   /* words per thread in the line scan (4) */
constexpr uint32_t DMAX = 64;       /* documents per sub-batch */
constexpr uint32_t QMAX = 1024;     /* owners per sub-batch */
constexpr uint32_t NSTAGE = 48;     /* marker owners whose tuples are staged in shared memory */
constexpr uint32_t STRIDE = 40;     /* staged tuples per marker owner */

/* DF_NONASCII: the document must be lexed sequentially by the Unicode lexer (invalid UTF-8 or Unicode white space,
 * or any non-ASCII byte when the caller does not do per-line Unicode lexing); DF_UNI: valid UTF-8 beyond ASCII, no
 * Unicode white space -- only the lines that contain such bytes need the Unicode lexer (two-stage pipeline) */
enum : uint32_t { DF_NONASCII = 1, DF_INTERACT = 2, DF_QOVERFLOW = 4, DF_UNI = 8, DF_EXACT_MASK = 7 };

/* owner record: bits 0..14 position of the first special ('+' lines) or of the comment start (plain
 * lines), bit 15 = marker line, bits 16..30 line start, bit 31 = plain line whose comment is "//" */
constexpr uint32_t OW_MARKER = 1u << 15, OW_SLASH2 = 1u << 31;
OBM_HD uint32_t ow_pos(uint32_t r) { return r & 0x7FFFu; }
OBM_HD uint32_t ow_ls(uint32_t r) { return (r >> 16) & 0x7FFFu; }

/* what the scan phases (P1..P4, owner classification) need; k1_scan stages exactly this */
struct SmemScan {
    alignas(16) uint8_t data[NW * 32];
    alignas(16) uint32_t nlw[NW];   /* bit i of word w: byte 32w+i is '\n' (or precedes a document start) */
    alignas(16) uint32_t spw[NW];   /* bit i of word w: byte 32w+i is '#', '+', or a '/' that may start "//" */
    uint16_t nlpre[NW];             /* number of nlw bits in words [0, w) */
    uint32_t naw[NW / 32];          /* bit w%32 of naw[w/32]: word w holds a byte >= 0x80 */
    uint32_t owner[QMAX];           /* owner records in position order */
    uint32_t dstart[DMAX + 1];      /* document start positions, buffer-relative; [nd] = end */
    uint32_t dflag[DMAX];
    uint32_t scan_tmp[NT / 32 + 1];
    uint32_t n_owners, n_markers_q; /* owners; marker owners in mlist */
    uint32_t nd;
    uint32_t lo_pos, hi_pos;        /* valid byte range of `data` */
};
/* the fused tile kernel (mode 2) additionally lexes, stages and resolves inside the CTA */
struct Smem : SmemScan {
    alignas(16) obm_tuple stage[NSTAGE * STRIDE];
    uint32_t ocnt[QMAX + 1];        /* tuple count of the owner; after the scan: exclusive prefix E[] */
    uint16_t mlist[QMAX];           /* dense list of marker owners (indices into owner[]) */
    uint16_t mslot[QMAX];           /* owner -> index in mlist (marker owners only) */
    uint8_t odoc[QMAX];             /* document (index in the sub-batch) of the owner */
    uint32_t dcnt[DMAX + 1];        /* tuples per document; after the scan: exclusive offsets */
    uint32_t dfirst[DMAX + 1];      /* first owner of each document */
};

/* ---- P2: classification ---------------------------------------------------------------------- */
/* 4-bit mask: bit b set iff byte b of t is zero (t's bytes must be < 0x80) */
OBM_HD uint32_t zero_bytes4(uint32_t t) {
    uint32_t ne = ((t + 0x7F7F7F7Fu) >> 7) & 0x01010101u; /* 1 per non-zero byte */
    uint32_t eq = ne ^ 0x01010101u;
    return (eq * 0x00204081u >> 21) & 0xFu;
}

/* the same for any byte values */
OBM_HD uint32_t zero_bytes4_exact(uint32_t t) {
    const uint32_t z = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t) & 0x80808080u;
    return ((z >> 7) * 0x00204081u >> 21) & 0xFu;
}
OBM_HD void classify_word(SmemScan &S, uint32_t wi) {
    const uint32_t *src = reinterpret_cast<const uint32_t *>(S.data) + wi * 8;
    uint32_t nl = 0, hp = 0, sl = 0, hi = 0;
#if defined(__CUDA_ARCH__)
    const uint4 a = reinterpret_cast<const uint4 *>(src)[0], b = reinterpret_cast<const uint4 *>(src)[1];
    const uint32_t x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#else
    const uint32_t *x = src;
#endif
#pragma unroll
    for (int k = 0; k < 8; k++) {
        uint32_t v = x[k];
        hi |= v;
        nl |= zero_bytes4(v ^ 0x0A0A0A0Au) << (4 * k);
        hp |= zero_bytes4((v & 0xF7F7F7F7u) ^ 0x23232323u) << (4 * k); /* '#' (0x23) or '+' (0x2B) */
        sl |= zero_bytes4(v ^ 0x2F2F2F2Fu) << (4 * k);                  /* '/' */
    }
    if (hi & 0x80808080u) {
        /* bytes >= 0x80 in this word: the carry-free byte test above is only exact for 7-bit input -- redo the word with
         * the exact form (the bitmaps of such words now matter: valid UTF-8 documents stay on the line-parallel path) */
        nl = hp = sl = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const uint32_t v = x[k];
            nl |= zero_bytes4_exact(v ^ 0x0A0A0A0Au) << (4 * k);
            hp |= zero_bytes4_exact((v & 0xF7F7F7F7u) ^ 0x23232323u) << (4 * k);
            sl |= zero_bytes4_exact(v ^ 0x2F2F2F2Fu) << (4 * k);
        }
    }
    /* specials: the bytes that can start a comment or a marker in state lex / lexComment (state.go:20-33,48):
     * '#', '+', and a '/' followed by another '/' (the word's last byte cannot see its successor: kept) */
    const uint32_t sp = hp | (sl & ((sl >> 1) | 0x80000000u));
    /* keep only bytes inside [lo_pos, hi_pos) */
    uint32_t w0 = wi * 32;
    uint32_t keep = 0xFFFFFFFFu;
    if (S.lo_pos > w0) keep &= (S.lo_pos - w0 >= 32) ? 0u : (0xFFFFFFFFu << (S.lo_pos - w0));
    if (S.hi_pos < w0 + 32) keep &= (S.hi_pos <= w0) ? 0u : (0xFFFFFFFFu >> (w0 + 32 - S.hi_pos));
    S.nlw[wi] = nl & keep;
    S.spw[wi] = sp & keep;
    bool na = (hi & 0x80808080u) != 0 && keep != 0;
#if defined(__CUDA_ARCH__)
    uint32_t bal = __ballot_sync(0xFFFFFFFFu, na); /* callers keep warps converged and wi = base + lane */
    if ((wi & 31) == 0) S.naw[wi >> 5] = bal;
#else
    if ((wi & 31) == 0) S.naw[wi >> 5] = 0;
    if (na) S.naw[wi >> 5] |= 1u << (wi & 31);
#endif
}

OBM_HD void atomic_or_u32(uint32_t *p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}
OBM_HD uint32_t atomic_inc_u32(uint32_t *p) {
#if defined(__CUDA_ARCH__)
    return atomicAdd(p, 1u);
#else
    return (*p)++;
#endif
}

/* ---- P3: per-document preparation (thread d < nd) ---------------------------------------------- */
/* Go's utf8.DecodeRune validity (no overlongs, no surrogates, <= U+10FFFF) over bytes [q, e) of S.data, plus: no
 * code point of unicode.IsSpace beyond ASCII (U+0085, U+00A0, U+1680, U+2000-200A, U+2028, U+2029, U+202F, U+205F,
 * U+3000).  Why both: an invalid byte makes the reference discard 3 bytes for 1 (discard.go:27-30) and Unicode white
 * space is skipped by peekedWhitespaced / consumed as `width` RUNES (peek.go:65-89, consume.go:39-41) -- either can
 * reach across a newline from a line that owns no tuple, so such documents are lexed sequentially.  Valid text
 * without them keeps every line independent (SURVEY.md A.11): only ASCII white space separates tokens. */
OBM_FN bool utf8_plain(const SmemScan &S, uint32_t q, uint32_t e) {
    uint32_t p = q;
    while (p < e) {
        const uint32_t w = p >> 5;
        if (!((S.naw[w >> 5] >> (w & 31)) & 1u)) { p = (w + 1) << 5; continue; } /* all-ASCII word */
        const uint32_t wend = ((w + 1) << 5) < e ? ((w + 1) << 5) : e;
        while (p < wend) {
            const uint32_t b0 = S.data[p];
            if (b0 < 0x80) { p++; continue; }
            uint32_t need, lo = 0x80, hi = 0xBF;
            if (b0 >= 0xC2 && b0 <= 0xDF) need = 1;
            else if (b0 >= 0xE0 && b0 <= 0xEF) { need = 2; if (b0 == 0xE0) lo = 0xA0; if (b0 == 0xED) hi = 0x9F; }
            else if (b0 >= 0xF0 && b0 <= 0xF4) { need = 3; if (b0 == 0xF0) lo = 0x90; if (b0 == 0xF4) hi = 0x8F; }
            else return false;
            if (p + need >= e) return false; /* truncated at the end of the document */
            const uint32_t b1 = S.data[p + 1];
            if (b1 < lo || b1 > hi) return false;
            uint32_t b2 = 0, b3 = 0;
            if (need >= 2) { b2 = S.data[p + 2]; if (b2 < 0x80 || b2 > 0xBF) return false; }
            if (need == 3) { b3 = S.data[p + 3]; if (b3 < 0x80 || b3 > 0xBF) return false; }
            /* Unicode white space */
            if (b0 == 0xC2 && (b1 == 0x85 || b1 == 0xA0)) return false;
            if (b0 == 0xE1 && b1 == 0x9A && b2 == 0x80) return false;
            if (b0 == 0xE2 && b1 == 0x80 && (b2 <= 0x8A || b2 == 0xA8 || b2 == 0xA9 || b2 == 0xAF)) return false;
            if (b0 == 0xE2 && b1 == 0x81 && b2 == 0x9F) return false;
            if (b0 == 0xE3 && b1 == 0x80 && b2 == 0x80) return false;
            p += need + 1;
        }
    }
    return true;
}
/* uni_lines: the caller lexes lines with non-ASCII bytes one by one with the Unicode lexer (two-stage pipeline);
 * otherwise any byte >= 0x80 sends the whole document to the sequential path (fused kernel) */
OBM_FN void doc_prep(SmemScan &S, uint32_t d, bool uni_lines = false) {
    uint32_t q = S.dstart[d], e = S.dstart[d + 1];
    if (q > S.lo_pos) atomic_or_u32(&S.nlw[(q - 1) >> 5], 1u << ((q - 1) & 31)); /* virtual newline before the document */
    uint32_t flag = 0;
    if (e > q) {
        uint32_t w0 = q >> 5, w1 = (e - 1) >> 5; /* words touched, boundary words included (conservative) */
        for (uint32_t g = w0 >> 5; g <= (w1 >> 5); g++) {
            uint32_t m = S.naw[g];
            uint32_t lo = g * 32, hiw = lo + 31;
            if (w0 > lo) m &= 0xFFFFFFFFu << (w0 - lo);
            if (w1 < hiw) m &= 0xFFFFFFFFu >> (hiw - w1);
            if (m) { flag = DF_NONASCII; break; }
        }
        if (flag && uni_lines && utf8_plain(S, q, e)) flag = DF_UNI;
    }
    S.dflag[d] = flag;
}

/* ---- P4: line scan (thread t owns words [WPT*t, WPT*t+WPT)) -------------------------------------- */
/* first position >= from whose (sp|nl) bit is set, or hi_pos if none */
OBM_FN uint32_t next_event(const SmemScan &S, uint32_t from) {
    if (from >= S.hi_pos) return S.hi_pos;
    uint32_t w = from >> 5;
    uint32_t m = (S.spw[w] | S.nlw[w]) & (0xFFFFFFFFu << (from & 31));
    const uint32_t wend = (S.hi_pos + 31) >> 5;
    while (m == 0) {
        if (++w >= wend) return S.hi_pos;
        m = S.spw[w] | S.nlw[w];
    }
    uint32_t pos = w * 32 + OBMT_CTZ(m);
    return pos < S.hi_pos ? pos : S.hi_pos;
}
OBM_HD bool is_sp(const SmemScan &S, uint32_t pos) { return (S.spw[pos >> 5] >> (pos & 31)) & 1u; }
OBM_HD bool is_nl(const SmemScan &S, uint32_t pos) { return (S.nlw[pos >> 5] >> (pos & 31)) & 1u; }

/* ---- P4a: which lines have a special byte, bit-parallel -------------------------------------------
 * A line starts right after every newline bit (and at lo_pos).  Let X = nl|sp be the "event" bits and
 * M the line-start bits.  Adding M to ~X lets each start bit ripple through the non-event bytes until it
 * lands on the line's first event; (~X + M) & X therefore marks the FIRST event of every line, and
 * & sp keeps the lines whose first event is a special byte -- those lines get an owner.  The carry
 * that leaves a word (a line with no event yet) enters the next word; across threads and warps it is
 * resolved with generate/propagate look-ahead (carry_lookahead32). */
struct LineBits { uint32_t own[WPT]; uint32_t n_own, n_nl; };

/* this thread's four words with carry-in `cin`; returns the carry out */
OBM_HD uint32_t first_events(const uint32_t (&nl)[WPT], const uint32_t (&sp)[WPT], const uint32_t (&m)[WPT], uint32_t cin, LineBits *lb) {
    uint32_t c = cin;
#pragma unroll
    for (uint32_t j = 0; j < WPT; j++) {
        uint32_t x = nl[j] | sp[j];
        uint64_t s = (uint64_t)(~x) + m[j] + c;
        c = (uint32_t)(s >> 32);
        if (lb) lb->own[j] = (uint32_t)s & x & sp[j];
    }
    return c;
}
/* line-start bits of the thread's words: after every newline, plus the buffer's first byte */
OBM_HD void line_starts(const SmemScan &S, uint32_t t, const uint32_t (&nl)[WPT], uint32_t (&m)[WPT]) {
    uint32_t prev = t ? (S.nlw[t * WPT - 1] >> 31) : 0u;
#pragma unroll
    for (uint32_t j = 0; j < WPT; j++) {
        m[j] = (nl[j] << 1) | prev;
        prev = nl[j] >> 31;
        uint32_t w = t * WPT + j;
        if (S.lo_pos < S.hi_pos && (S.lo_pos >> 5) == w) m[j] |= 1u << (S.lo_pos & 31);
    }
}
/* 32 carry chains in one add: lane i generates (G bit) or propagates (P bit, disjoint from G) a carry.
 * Returns the mask of lanes that RECEIVE a carry; *cout = carry out of lane 31. */
OBM_HD uint32_t carry_lookahead32(uint32_t G, uint32_t P, uint32_t cin, uint32_t *cout) {
    uint64_t s = (uint64_t)(G | P) + G + cin;
    *cout = (uint32_t)(s >> 32);
    return (uint32_t)s ^ P; /* sum ^ a ^ b with a = G|P, b = G, a ^ b = P */
}

/* previous line start: position after the last newline bit below `pos` (or lo_pos) */
OBM_FN uint32_t line_start_of(const SmemScan &S, uint32_t pos) {
    uint32_t w = pos >> 5;
    uint32_t m = S.nlw[w] & ((1u << (pos & 31)) - 1u);
    const uint32_t wlo = S.lo_pos >> 5;
    while (m == 0) {
        if (w == wlo) return S.lo_pos;
        m = S.nlw[--w];
    }
#if defined(__CUDA_ARCH__)
    uint32_t top = 31u - (uint32_t)__clz((int)m);
#else
    uint32_t top = 31u - (uint32_t)__builtin_clz(m);
#endif
    uint32_t ls = w * 32 + top + 1;
    return ls > S.lo_pos ? ls : S.lo_pos;
}

constexpr uint32_t OW_NONE = 0xFFFFFFFFu; /* not a valid record: it would be a MARKER line that is also flagged "//" */
/* Classifies the line whose first special byte is at `first`: marker line, plain comment line, or a line
 * that produces no tuple (OW_NONE).  A position carrying both bits (virtual newline on a document's
 * last byte) is a special that also ends the line. */
OBM_FN uint32_t classify_line(const SmemScan &S, uint32_t first, uint32_t start) {
    uint32_t ev = first;
    uint32_t comment = 0xFFFFFFFFu; bool slash2 = false;
    for (;;) {
        uint32_t c = S.data[ev];
        if (c == '+') return first | OW_MARKER | (start << 16);
        if (comment == 0xFFFFFFFFu) {
            if (c == '#') comment = ev;
            else if (c == '/' && ev + 1 < S.hi_pos && S.data[ev + 1] == '/' && !is_nl(S, ev)) { comment = ev; slash2 = true; }
        }
        if (is_nl(S, ev)) break; /* the special sits on the line's last byte */
        ev = next_event(S, ev + 1);
        if (ev >= S.hi_pos || !is_sp(S, ev)) break;
    }
    if (comment == 0xFFFFFFFFu) return OW_NONE;
    return comment | (start << 16) | (slash2 ? OW_SLASH2 : 0u);
}

/* number of nlw bits at positions < q */
OBM_HD uint32_t nl_before(const SmemScan &S, uint32_t q) {
    uint32_t w = q >> 5;
    if (w >= NW) return (uint32_t)S.nlpre[NW - 1] + OBMT_POPC(S.nlw[NW - 1]);
    return (uint32_t)S.nlpre[w] + OBMT_POPC(S.nlw[w] & ((1u << (q & 31)) - 1u));
}

/* ---- P5 / P7: owners ------------------------------------------------------------------------- */
struct BitmapAccel {
    const SmemScan *S; uint32_t dpos, dend; /* document start / end, buffer-relative */
    OBM_HD uint32_t next_interesting(uint32_t p) const {
        uint32_t q = next_event(*S, dpos + p);
        if (q > dend) q = dend;
        return q - dpos;
    }
};

/* document (index in the sub-batch) containing buffer position `pos`: the last d with dstart[d] <= pos */
OBM_FN uint32_t doc_of(const SmemScan &S, uint32_t pos) {
    uint32_t lo = 0, hi = S.nd;
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (S.dstart[mid] <= pos) lo = mid; else hi = mid;
    }
    return lo;
}

/* The two lexer instantiations the tile kernel carries, each compiled once (noinline). */
typedef obm::Lexer<obm::SmallSink, BitmapAccel, true, const uint8_t *, true> LineLexer;
typedef obm::Lexer<obm::SmallSink, obm::NoAccel, false, const uint8_t *, true> DocLexer;

/* marker line: LINE mode from the first special.  Sink and lexer live in registers (everything inlines
 * into this one function, which is compiled once and called from the stage and fill phases). */
struct LineResult { uint32_t tuples, markers, lexemes; bool interact; };
OBM_HD_NOINLINE LineResult run_marker_line(const Smem &S, const obm::Tables &T, uint32_t rec, uint32_t d, obm_tuple *out, uint32_t cap) {
    uint32_t first = ow_pos(rec), ls = ow_ls(rec);
    uint32_t dpos = S.dstart[d], dend = S.dstart[d + 1];
    uint32_t line = 1 + nl_before(S, ls) - nl_before(S, dpos);
    BitmapAccel acc{&S, dpos, dend};
    obm::SmallSink sink(out, cap);
    LineLexer lx(T, S.data + dpos, dend - dpos, sink, first - dpos, line, ls - dpos, !(line == 1 && ls == dpos), acc);
    lx.fill_windows(lx.p);
    int st = lx.run<true>();
    uint32_t end_line = lx.line_p - (st == obm::RUN_LINE_END ? 1u : 0u);
    LineResult r;
    r.tuples = sink.n_tuples; r.markers = sink.n_markers; r.lexemes = sink.n_lexemes;
    r.interact = (st == obm::RUN_FATAL) || (end_line != line);
    return r;
}
/* whole document through the exact (Unicode) lexer */
OBM_HD_NOINLINE int run_doc_exact(const Smem &S, const obm::Tables &T, uint32_t d, obm::SmallSink &sink) {
    uint32_t dpos = S.dstart[d], dend = S.dstart[d + 1];
    DocLexer lx(T, S.data + dpos, dend - dpos, sink);
    return lx.run<false>();
}

/* plain line: [LINE] Comment.  Returns the tuple count; writes when out != nullptr. */
OBM_FN uint32_t plain_line(const Smem &S, uint32_t rec, uint32_t d, obm_tuple *out, uint64_t room) {
    uint32_t cpos = ow_pos(rec), ls = ow_ls(rec), dpos = S.dstart[d];
    bool need_line = true;
    uint32_t line = 0;
    if (ls == dpos) need_line = false;          /* first line of the document: basis (1, 0) is implied */
    uint32_t k = 0;
    if (out) {
        if (need_line) {
            line = 1 + nl_before(S, ls) - nl_before(S, dpos);
            if (line >> OBM_LEN_BITS) { if (k < room) out[k] = OBM_TUPLE(OBM_K_LINEHI, line >> OBM_LEN_BITS, 0); k++; }
            if (k < room) out[k] = OBM_TUPLE(OBM_K_LINE, ls - dpos, line & OBM_MAX_LEN);
            k++;
        }
        if (k < room) out[k] = OBM_TUPLE(OBM_K_COMMENT, cpos - dpos, (rec & OW_SLASH2) ? 2 : 1);
        k++;
        return k;
    }
    return need_line ? 2u : 1u; /* line numbers inside a <= 16 KiB document never need LINEHI */
}

/* P5a body for owner o (every line that has a special byte): S.owner[o] holds the position of the line's
 * first special; classify the line, find its document, count plain lines, compact marker lines.
 * odoc bit 7 marks a line that produces no tuple. */
OBM_FN void owner_prepare(Smem &S, uint32_t o) {
    uint32_t first = S.owner[o];
    uint32_t ls = line_start_of(S, first);
    uint32_t d = doc_of(S, ls);
    uint32_t rec = S.dflag[d] ? OW_NONE : classify_line(S, first, ls);
    if (rec == OW_NONE) { S.owner[o] = first | (ls << 16); S.odoc[o] = (uint8_t)(d | 0x80u); S.ocnt[o] = 0; return; }
    S.owner[o] = rec;
    S.odoc[o] = (uint8_t)d;
    if (rec & OW_MARKER) {
        uint32_t m = atomic_inc_u32(&S.n_markers_q);
        S.mlist[m] = (uint16_t)o; S.mslot[o] = (uint16_t)m;
        S.ocnt[o] = 0;
    } else {
        S.ocnt[o] = plain_line(S, rec, d, nullptr, 0);
    }
}

/* P5b body for marker owner m (dense): tokenize, stage */
OBM_FN void marker_stage(Smem &S, const obm::Tables &T, uint32_t m) {
    uint32_t o = S.mlist[m];
    uint32_t d = S.odoc[o]; /* marker owners never carry the dead flag */
    if (S.dflag[d]) { S.ocnt[o] = 0; return; }
    LineResult r = run_marker_line(S, T, S.owner[o], d, m < NSTAGE ? S.stage + m * STRIDE : nullptr, m < NSTAGE ? STRIDE : 0u);
    S.ocnt[o] = r.tuples;
    if (r.interact) atomic_or_u32(&S.dflag[d], DF_INTERACT);
}

/* first owner whose line start is >= pos */
OBM_FN uint32_t first_owner_at(const Smem &S, uint32_t pos) {
    uint32_t lo = 0, hi = S.n_owners;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (ow_ls(S.owner[mid]) < pos) lo = mid + 1; else hi = mid;
    }
    return lo;
}

/* P6 body for document d (after the owner-count scan turned ocnt[] into E[]): tuples of the document */
OBM_FN void doc_count(Smem &S, const obm::Tables &T, uint32_t d) {
    if (S.dflag[d]) { /* exact path, sequential, same core */
        obm::SmallSink sink(nullptr, 0);
        run_doc_exact(S, T, d, sink);
        S.dcnt[d] = sink.n_tuples;
    } else {
        S.dcnt[d] = S.ocnt[S.dfirst[d + 1]] - S.ocnt[S.dfirst[d]] + 1; /* + EOF */
    }
}

struct FillStats { uint32_t markers, lexemes, exact_docs, fatal_docs; };

/* global tuple index of owner o's first tuple */
OBM_HD uint64_t owner_at(const Smem &S, uint32_t o, uint64_t batch_base) {
    uint32_t d = S.odoc[o] & 0x7Fu;
    return batch_base + S.dcnt[d] + (S.ocnt[o] - S.ocnt[S.dfirst[d]]);
}

/* P7 body for owner o handled by ONE thread: plain lines, and marker lines that were not staged */
OBM_FN void owner_fill_thread(const Smem &S, const obm::Tables &T, uint32_t o, uint32_t cnt, obm_tuple *out, uint64_t out_cap,
                              uint64_t batch_base, FillStats &fs) {
    uint32_t d = S.odoc[o];
    if (d & 0x80u) return; /* the line produces no tuple */
    if (S.dflag[d]) return;
    uint32_t rec = S.owner[o];
    uint64_t at = owner_at(S, o, batch_base);
    uint64_t room = at < out_cap ? out_cap - at : 0;
    if (!(rec & OW_MARKER)) { plain_line(S, rec, d, out + at, room); fs.lexemes += 1; return; }
    uint32_t m = S.mslot[o];
    if (m < NSTAGE && cnt <= STRIDE) return; /* staged: copied by owner_fill_staged */
    LineResult r = run_marker_line(S, T, rec, d, out + at, room > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)room);
    fs.markers += r.markers; fs.lexemes += r.lexemes;
}

/* P7 body for staged marker owner m, lane `lane` of `nlanes` cooperating lanes */
OBM_FN void owner_fill_staged(const Smem &S, uint32_t m, uint32_t lane, uint32_t nlanes, obm_tuple *out, uint64_t out_cap,
                              uint64_t batch_base, FillStats &fs) {
    uint32_t o = S.mlist[m];
    uint32_t d = S.odoc[o];
    if (S.dflag[d]) return;
    uint32_t cnt = S.ocnt[o + 1] - S.ocnt[o]; /* E[] differences: owners are contiguous in E */
    if (cnt > STRIDE) return;
    uint64_t at = owner_at(S, o, batch_base);
    const obm_tuple *src = S.stage + m * STRIDE;
    for (uint32_t k = lane; k < cnt; k += nlanes) {
        obm_tuple t = src[k];
        if (at + k < out_cap) out[at + k] = t;
        uint32_t kind = OBM_TUPLE_KIND(t);
        fs.markers += (kind == OBM_K_MARKER_START);
        fs.lexemes += (kind <= OBM_K_EOF) || (kind >= OBM_K_WARN_NOSCOPE);
    }
}

/* P7 body for document d: EOF tuple of a regular document, or the whole irregular document */
OBM_FN void doc_fill(const Smem &S, const obm::Tables &T, uint32_t d, obm_tuple *out, uint64_t out_cap,
                     uint64_t batch_base, FillStats &fs) {
    uint64_t at = batch_base + S.dcnt[d];
    if (S.dflag[d]) {
        uint64_t room = at < out_cap ? out_cap - at : 0;
        obm::SmallSink sink(out + at, room > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)room);
        int st = run_doc_exact(S, T, d, sink);
        fs.markers += sink.n_markers; fs.lexemes += sink.n_lexemes; fs.exact_docs += 1; fs.fatal_docs += (st == obm::RUN_FATAL);
    } else {
        uint64_t eof_at = batch_base + S.dcnt[d + 1] - 1;
        if (eof_at < out_cap) out[eof_at] = OBM_TUPLE(OBM_K_EOF, S.dstart[d + 1] - S.dstart[d], 0);
        fs.lexemes += 1;
    }
}

} /* namespace obmt */
#endif
