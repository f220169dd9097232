/*
 * obm_pipe.h -- host/device logic of the two-stage pipeline (mode 0), on top of obm_tile.h:
 *
 *   K1 scan   per 16 KiB tile, shared-memory resident: TMA stage, classify, bit-parallel line scan, owner
 *             classification.  Emits compact work records to HBM instead of lexing: one 8-byte ITEM per line
 *             that owns tuples (position order inside a unit), an EOF item per document, a 16-byte unit record
 *   K2 units  one WARP per unit: marker items are lexed once (a lane per line) by the ASCII instantiation of
 *             obm::Lexer from a shared-memory copy of the line, tuples staged in shared memory; item counts ->
 *             unit total -> two-level decoupled look-back over units -> final positions -> write
 *
 * Why two kernels: in the fused tile kernel (obm_fast.cuh, mode 2) the marker phase is a long dependent chain
 * on a few warps while shared memory caps residency at 3 CTAs/SM and block barriers make every warp wait for
 * the slowest line.  Here K1 has no lexing and K2 has no block barrier.
 */
#ifndef OBM_PIPE_H
#define OBM_PIPE_H

#include "obm_tile.h"

namespace obmp {

using obmt::SmemScan;


/* ---- item: one line that owns tuples (8 bytes) ---------------------------------------------------
 *  bits  0..13  ls    line start, document-relative (documents on this path are <= 16,368 B)
 *  bits 14..27  pos   marker line: first special byte; plain line: comment start (document-relative)
 *  bits 28..41  line  line number (1-based)
 *  bit  42      marker line
 *  bit  43      plain line whose comment is "//"
 *  bit  44      dead (the line has specials but produces no tuple)
 *  bits 45..50  doc   document index inside the sub-batch (< DMAX = 64)
 *  (marker / EOF / LARGE items use the upper bits differently: see below) */
typedef uint64_t item_t;
OBM_HD item_t make_item(uint32_t ls, uint32_t pos, uint32_t line, bool marker, bool slash2, bool dead, uint32_t d) {
    return (item_t)ls | ((item_t)pos << 14) | ((item_t)line << 28) | ((item_t)marker << 42) | ((item_t)slash2 << 43) |
           ((item_t)dead << 44) | ((item_t)d << 45);
}
OBM_HD uint32_t it_ls(item_t i) { return (uint32_t)(i & 0x3FFF); }
OBM_HD uint32_t it_pos(item_t i) { return (uint32_t)((i >> 14) & 0x3FFF); }
OBM_HD uint32_t it_line(item_t i) { return (uint32_t)((i >> 28) & 0x3FFF); }
OBM_HD bool it_marker(item_t i) { return (i >> 42) & 1; }
OBM_HD bool it_slash2(item_t i) { return (i >> 43) & 1; }
OBM_HD bool it_dead(item_t i) { return !it_marker(i) && ((i >> 44) & 1); } /* marker items reuse bit 44 (it_unicode) */
OBM_HD uint32_t it_doc(item_t i) { return (uint32_t)((i >> 45) & 0x3F); }

/* K2 result per marker line */
OBM_HD uint32_t make_mres(uint32_t tuples, bool irregular) { return tuples | (irregular ? 0x80000000u : 0u); }
OBM_HD uint32_t mres_tuples(uint32_t r) { return r & 0x7FFFFFFFu; }
OBM_HD bool mres_irregular(uint32_t r) { return r >> 31; }

/* document flags (u32 per document) */
enum : uint32_t { GF_NONASCII = 1, GF_INTERACT = 2, GF_QOVERFLOW = 4, GF_LARGE = 8 };

/* ---- K2: one marker line straight from global memory -------------------------------------------- */
/* lex / lexComment skipping without bitmaps: the next byte in [p, line_end] that is '\n' or one of # ' + /
 * (same contract as obm::NoAccel but 4 bytes per step on the aligned words of the line) */
template <class Src>
struct LineAccelT {
    Src d; uint32_t line_end;
    OBM_HD uint32_t next_interesting(uint32_t p) const {
        while (p < line_end) {
            uint32_t mis = obm::src_mis(d, p);
            uint32_t w = obm::src_ldw(d, (int32_t)p - (int32_t)mis);
            /* exact form: the aligned word may hold bytes >= 0x80 of a NEIGHBOURING document below p, whose carries would hide a match */
            uint32_t sp = obmt::zero_bytes4_exact((w & 0xF3F3F3F3u) ^ 0x23232323u) >> mis;
            if (sp) {
#if defined(__CUDA_ARCH__)
                uint32_t q = p + (uint32_t)(__ffs((int)sp) - 1);
#else
                uint32_t q = p + (uint32_t)__builtin_ctz(sp);
#endif
                return q < line_end ? q : line_end;
            }
            p += 4 - mis;
        }
        return line_end;
    }
};
typedef LineAccelT<const uint8_t *> LineAccel;
template <class Src> using GLineLexerT = obm::Lexer<obm::SmallSink, LineAccelT<Src>, true, Src, true>;
typedef GLineLexerT<const uint8_t *> GLineLexer;

OBM_HD uint32_t plain_count_fwd(item_t it) { return it_line(it) == 1 ? 1u : 2u; }

/* ==== two-stage pipeline (mode 0): K1 emits per-unit item runs, K2 lexes + assembles one unit per warp ====
 * Within a unit the items are in position order.  Besides one item per tuple-owning line, every document
 * closes with an EOF item, so tuple positions are a plain prefix sum over item counts.  A marker item
 * carries everything K2 needs to lex its line (there is no separate marker-line list):
 *   marker item : ls | first<<14 | line<<28 | 1<<42 | line_end[13]<<43 | doc6<<45 | line_end[0..12]<<51
 *   plain item  : ls | comment<<14 | line<<28 | slash2<<43 | dead<<44 | doc6<<45
 *   EOF item    : doc length | doc6<<45 | 1<<51 | exact<<52      (exact: K1 flagged the document)
 *   LARGE item  : 1<<51 | 1<<53                                  (document = last of the unit; > MAXDOC)
 * A unit is one K1 sub-batch (<= DMAX whole documents of one tile, <= QMAX owning lines); unit ids are
 * static and in document order, so a decoupled look-back over units orders the output. */
OBM_HD item_t make_marker_item(uint32_t ls, uint32_t first, uint32_t line, uint32_t d, uint32_t line_end) {
    return (item_t)ls | ((item_t)first << 14) | ((item_t)line << 28) | ((item_t)1 << 42) | ((item_t)((line_end >> 13) & 1u) << 43) |
           ((item_t)d << 45) | ((item_t)(line_end & 0x1FFFu) << 51);
}
OBM_HD bool it_unicode(item_t i) { return it_marker(i) && ((i >> 44) & 1); } /* lexed from the line start by the Unicode lexer */
OBM_HD uint32_t it_line_end(item_t i) { return (uint32_t)((i >> 51) & 0x1FFF) | ((uint32_t)((i >> 43) & 1) << 13); }
OBM_HD item_t make_eof_item(uint32_t len, uint32_t d, bool exact) { return (item_t)len | ((item_t)d << 45) | ((item_t)1 << 51) | ((item_t)exact << 52); }
OBM_HD item_t make_large_item() { return ((item_t)1 << 51) | ((item_t)1 << 53); }
OBM_HD bool it_eof(item_t i) { return !it_marker(i) && ((i >> 51) & 1); }
OBM_HD bool it_exact(item_t i) { return !it_marker(i) && ((i >> 52) & 1); }
OBM_HD bool it_large(item_t i) { return !it_marker(i) && ((i >> 53) & 1); }

/* unit record (16 B): where the unit's items are, its first document, item / small-document counts */
struct Unit { uint64_t item_base; uint32_t doc_base; uint32_t n; /* n_items | nd << 16 */ };
OBM_HD uint32_t unit_items(const Unit &u) { return u.n & 0xFFFFu; }
OBM_HD uint32_t unit_nd(const Unit &u) { return u.n >> 16; }

/* per-tile record for K1 (written by k_tile_units): everything the tile loop needs before it can issue its first
 * TMA load, so that one 32-byte load replaces a chain of dependent ones and the next tile's load can be issued early */
struct TileRec { uint32_t d_first; uint32_t d_last; /* bit 31: the last document is large */ uint32_t pad0, pad1; uint64_t b0, b1; /* byte range of the first sub-batch */ };

constexpr uint32_t W_WARPS = 4;         /* warps per K2 CTA (each works alone) */
constexpr uint32_t W_MLCAP = 32;        /* marker lines staged per block = one per lane */
constexpr uint32_t W_LTS = 23;          /* staged tuples per marker line (odd stride: no bank clash) */
constexpr uint32_t W_POOL = 256;        /* 16-byte chunks of line text staged per warp (4 KiB) */
constexpr uint32_t W_LOOK = 24;         /* bytes staged past a line's newline: whitespace run + longest peeked token */
constexpr uint32_t W_TOKEN = 8;         /* >= the longest token a whitespace-skipping peek compares ("false") */
constexpr uint32_t W_ICAP = 256;        /* items of a unit handled as one block (larger units: 32-item blocks) */
constexpr uint16_t G_CNT_LOOKUP = 0xFFFF; /* item count lives in counts[doc] (exact / large documents) */

/* K1: owner o of the sub-batch -> item */
OBM_FN item_t k1_owner_item(const SmemScan &S, uint32_t o) {
    uint32_t first = S.owner[o];
    uint32_t ls = obmt::line_start_of(S, first);
    uint32_t d = obmt::doc_of(S, ls);
    uint32_t dpos = S.dstart[d], dend = S.dstart[d + 1];
    const uint32_t df = S.dflag[d];
    if (df & obmt::DF_EXACT_MASK) return make_item(ls - dpos, first - dpos, 0, false, false, true, d);
    if (df & obmt::DF_UNI) {
        /* valid UTF-8 document: a line with bytes >= 0x80 (judged per 32-byte word: conservative) is lexed as a whole
         * by the Unicode lexer, from its start; all-ASCII lines take the usual path */
        uint32_t e = first;
        for (;;) { if (e >= dend) { e = dend; break; } if (obmt::is_nl(S, e) && S.data[e] == '\n') break; e = obmt::next_event(S, e + 1); }
        const uint32_t last = e < S.hi_pos ? e : S.hi_pos - 1;
        bool na = false;
        for (uint32_t w = ls >> 5; w <= (last >> 5); w++) na |= ((S.naw[w >> 5] >> (w & 31)) & 1u) != 0;
        if (na) {
            const uint32_t line = 1 + obmt::nl_before(S, ls) - obmt::nl_before(S, dpos);
            return make_marker_item(ls - dpos, ls - dpos, line, d, e - dpos) | ((item_t)1 << 44);
        }
    }
    uint32_t rec = obmt::classify_line(S, first, ls);
    if (rec == obmt::OW_NONE) return make_item(ls - dpos, first - dpos, 0, false, false, true, d);
    uint32_t line = 1 + obmt::nl_before(S, ls) - obmt::nl_before(S, dpos);
    if (!(rec & obmt::OW_MARKER)) return make_item(ls - dpos, obmt::ow_pos(rec) - dpos, line, false, (rec & obmt::OW_SLASH2) != 0, false, d);
    uint32_t e = first;
    for (;;) { if (e >= dend) { e = dend; break; } if (obmt::is_nl(S, e) && S.data[e] == '\n') break; e = obmt::next_event(S, e + 1); }
    return make_marker_item(ls - dpos, first - dpos, line, d, e - dpos);
}

/* K2: a line of a valid-UTF-8 document that contains bytes >= 0x80: the Unicode lexer in LINE mode from the line
 * start, straight from global memory.  Regular iff it stopped exactly behind this line's newline. */
typedef obm::Lexer<obm::SmallSink, obm::NoAccel, false, const uint8_t *, true> GUniLexer;
OBM_HD_NOINLINE uint32_t k2_unicode_item(const obm::Tables &T, const uint8_t *doc, uint32_t n, item_t it, obm_tuple *out, uint32_t cap,
                                         uint32_t *markers = nullptr, uint32_t *lexemes = nullptr) {
    const uint32_t ls = it_ls(it), line = it_line(it), le = it_line_end(it);
    obm::SmallSink sink(out, cap);
    GUniLexer lx(T, doc, n, sink, ls, line, ls, !(line == 1 && ls == 0));
    const int st = lx.run<true>();
    const uint32_t end_line = lx.line_p - (st == obm::RUN_LINE_END ? 1u : 0u);
    const bool regular = st != obm::RUN_FATAL && end_line == line &&
                         (st == obm::RUN_LINE_END ? lx.p == le + 1u : (le == n && lx.p == n));
    if (markers) *markers += sink.n_markers;
    if (lexemes) *lexemes += sink.n_lexemes;
    return make_mres(sink.n_tuples, !regular);
}

/* K2: lex the line of a marker item of document doc[0..n) (global memory) */
template <class Src>
OBM_HD_NOINLINE uint32_t k2_marker_item(const obm::Tables &T, Src doc, uint32_t n, item_t it, obm_tuple *out, uint32_t cap,
                                        uint32_t *markers = nullptr, uint32_t *lexemes = nullptr) {
    const uint32_t ls = it_ls(it), first = it_pos(it), line = it_line(it);
    LineAccelT<Src> acc{doc, it_line_end(it)};
    obm::SmallSink sink(out, cap);
    GLineLexerT<Src> lx(T, doc, n, sink, first, line, ls, !(line == 1 && ls == 0), acc);
    lx.fill_windows(lx.p);
    int st = lx.template run<true>();
    uint32_t end_line = lx.line_p - (st == obm::RUN_LINE_END ? 1u : 0u);
    bool irregular = (st == obm::RUN_FATAL) || (end_line != line);
    if (markers) *markers += sink.n_markers;
    if (lexemes) *lexemes += sink.n_lexemes;
    return make_mres(sink.n_tuples, irregular);
}

/* ---- staged line text ------------------------------------------------------------------------------
 * K2 copies a marker line (first special byte .. newline + W_LOOK bytes, 16-byte chunks at the global
 * alignment) into shared memory and lexes it from there: all chunk loads of a warp are in flight at once
 * instead of one dependent miss per sector.  The lexer is handed a document pointer rebased onto the copy
 * and a document length cut at the end of the copy (`n_view`); that is exact as long as nothing past the
 * copy can matter:
 *   - bytes are only CONSUMED past the newline by constructs that make the line irregular (the document is
 *     then re-lexed exactly, whatever was read);
 *   - bytes are only PEEKED past the newline by whitespace-skipping token checks (peek.go:65-89: "true",
 *     "false", "//", "#"), which stop at the first non-whitespace byte + the token length.
 * line_view_safe() checks the second condition on the staged bytes; lines that fail it (or do not fit)
 * are lexed from global memory. */
struct LineView { uintptr_t g0, g1; uint32_t nch; };   /* staged address range [g0, g1), 16-byte chunks */
OBM_HD LineView line_view(const uint8_t *gdoc, uint32_t len, item_t it, const uint8_t *bytes, uint64_t total_bytes) {
    LineView v;
    const uintptr_t a_first = (uintptr_t)(gdoc + it_pos(it));
    uint32_t e = it_line_end(it) + 1u + W_LOOK; if (e > len) e = len;
    const uintptr_t lim = ((uintptr_t)(bytes + total_bytes) + 15u) & ~(uintptr_t)15u; /* readable end of the batch (obmarkers.h) */
    uintptr_t g1 = ((uintptr_t)(gdoc + e) + 15u) & ~(uintptr_t)15u; if (g1 > lim) g1 = lim;
    v.g0 = a_first & ~(uintptr_t)15u; v.g1 = g1; v.nch = (uint32_t)((g1 - v.g0) >> 4);
    return v;
}
/* sm: the staged copy of [g0, g1).  Returns n_view (> 0) when lexing from the copy is exact, else 0. */
OBM_HD uint32_t line_view_safe(const uint8_t *sm, const LineView &v, const uint8_t *gdoc, uint32_t len, item_t it) {
    const uintptr_t endrel = v.g1 - (uintptr_t)gdoc;
    const uint32_t n_view = endrel < len ? (uint32_t)endrel : len;
    if (n_view == len) return n_view;                      /* the copy reaches the real end of the document */
    uint32_t w = it_line_end(it) + 1u;                     /* first byte after the newline */
    const uint8_t *base = sm + (intptr_t)((uintptr_t)gdoc - v.g0); /* base[p] = document byte p (wraps: g0 is usually past gdoc) */
    while (w < n_view && obm::is_space(base[w])) w++;
    return (w + W_TOKEN <= n_view) ? n_view : 0u;
}

/* tuples of a non-marker item of a regular document */
OBM_HD uint32_t simple_count(item_t it) { return it_dead(it) ? 0u : it_eof(it) ? 1u : plain_count_fwd(it); }

/* ---- K3 ------------------------------------------------------------------------------------------ */
/* tuples of a plain item: [LINE] Comment */
OBM_HD uint32_t plain_count(item_t it) { return it_line(it) == 1 ? 1u : 2u; }
OBM_HD void plain_write(item_t it, obm_tuple *out, uint64_t at, uint64_t cap) {
    uint32_t k = 0;
    if (it_line(it) != 1) { if (at < cap) out[at] = OBM_TUPLE(OBM_K_LINE, it_ls(it), it_line(it)); k = 1; }
    if (at + k < cap) out[at + k] = OBM_TUPLE(OBM_K_COMMENT, it_pos(it), it_slash2(it) ? 2 : 1);
}

/* whole document through the exact (Unicode) lexer, from global memory: line after line in LINE mode plus the EOF
 * tuple -- the composition tests/hostsim checks against the whole-document run (hs_lex_doc_by_lines).  Written this
 * way so that K2 carries ONE instantiation of the Unicode lexer's run loop (run<true>, shared with k2_unicode_item):
 * a second one costs ~280 KB of code and showed up as instruction-cache misses in the hot ASCII path. */
OBM_HD_NOINLINE int doc_exact(const obm::Tables &T, const uint8_t *doc, uint32_t n, obm::SmallSink &sink) {
    uint32_t pos = 0, line = 1;
    while (pos < n) {
        GUniLexer lx(T, doc, n, sink, pos, line, pos, !(line == 1 && pos == 0));
        const int st = lx.run<true>();
        if (st == obm::RUN_FATAL) return obm::RUN_FATAL;
        if (st == obm::RUN_EOF) break;
        pos = lx.p; line = lx.line_p;
    }
    sink.put(OBM_K_EOF, n, 0);
    return obm::RUN_EOF;
}

} /* namespace obmp */
#endif
