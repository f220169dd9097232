/*
 * obm_warp_core.h -- the body of the fused warp kernel (see obm_warp.h), written against a small set of warp
 * collectives so that the very same source runs on the device (obm_warp.cuh: CUDA intrinsics) and, for logic
 * tests, on the host (tests/hostsim/warp_emu.h: 32 fibers in lock step).  The includer defines, before
 * including this file:
 *     WLANE()                lane id 0..31
 *     WBALLOT(pred)          __ballot_sync
 *     WSHFL(v, src)          __shfl_sync (u32), WSHFL_UP(v, delta)
 *     WSYNC()                __syncwarp (also orders the warp's shared-memory accesses)
 *     WTEXT(S)               the byte source of the staged text (ShBytes on the device, pointer on the host)
 *     WATOMIC_OR(p, v)       atomicOr on shared memory
 * and supplies a Hooks type with
 *     stage(W, gsrc, nbytes) bring nbytes (multiple of 16) from the 16-byte aligned global address gsrc into W.text
 *     stage_wait(W, nbytes)  ... and wait for them
 * The look-back chain over the units' tuple counts is driven by the caller between compute_unit and write_unit.
 */
#ifndef OBM_WARP_CORE_H
#define OBM_WARP_CORE_H

#include "obm_warp.h"

#ifndef OBMW_STAT
#define OBMW_STAT(name) ((void)0) /* the host replay counts how lines were lexed */
#endif
#if defined(__CUDACC__)
#define OBMW_DEV __device__ __forceinline__
#else
#define OBMW_DEV inline
#endif

namespace obmw {

/* ---- OBMW_PHASE_CLOCKS (a separate device build, libobmarkers_phase.so): k_warp_scan adds the cycles between phase
 * borders into per-warp registers and sums them over the warps at kernel end (tools/phase_cycles.py).  Off, the
 * macros below are empty and the kernels compile as without them. ---- */
enum : uint32_t { PC_STAGE, PC_A, PC_B, PC_C, PC_ASM, PC_AFIN, PC_WRITE, PC_CHAIN, PC_OTHER, PC_N };
#if defined(OBMW_PHASE_CLOCKS) && defined(__CUDACC__)
struct PhaseClk { uint32_t t0; uint32_t c[PC_N]; }; /* low 32 bits of clock64(): a warp's share of one launch stays far below 2^32 cycles */
#define OBMW_PC_PARAM , PhaseClk &pc
#define OBMW_PC_ARG , pc
#define OBMW_PC_MARK(b) do { const uint32_t t_ = (uint32_t)clock64(); pc.c[(b)] += t_ - pc.t0; pc.t0 = t_; } while (0)
#else
#define OBMW_PC_PARAM
#define OBMW_PC_ARG
#define OBMW_PC_MARK(b) ((void)0)
#endif

/* scratch of the unit being scanned */
struct UnitSet {
    union {
        struct { uint32_t nlw[NWORDS]; uint32_t spw[NWORDS]; } bm; /* phases A, B */
        struct { uint32_t stage[MLCAP * LTS]; uint32_t mstat[MLCAP]; } c; /* phase C on (the bitmaps are dead by then); mstat: staged line =
                                                                    * markers | lexemes << 8 | tuples << 16; MS_NONE: not staged */
    } u;
    orec_t orec[OWN_CAP];       /* phase A: position of the line's first special; phase B: owner record */
    uint16_t opos[OWN_CAP];     /* tuples of the owner; after the assembly: its tuple position inside the unit */
    uint8_t mlist[OWN_CAP];     /* marker rank -> owner */
};
struct WarpSmem {
    alignas(16) uint8_t text[BUFB + 64];
    UnitSet set;
    uint32_t fin[FIN_CAP];      /* the unit's tuples, packed (st_pack), in final order: what the DEFERRED write needs -- a warp scans
                                 * its next unit while this unit's tuple count travels through the chain (obm_warp.cuh) */
    uint16_t nlpre[NWORDS / 2]; /* newline bits in words [0, 2k): every second word, the odd ones add their neighbour's count */
    uint32_t naw[NWORDS / 32 + 1]; /* per row: the 32-byte words that hold bytes >= 0x80 */
    uint32_t dstart[DMAX + 2];  /* document starts, buffer-relative; [nd] = end */
    uint32_t dflag[DMAX + 1];
    uint16_t dcnt[DMAX + 1];    /* exclusive tuple offsets of the documents inside the unit */
    uint16_t dfo[DMAX + 2];     /* first owner of the document */
    alignas(8) uint64_t mbar;
};
static_assert(sizeof(uint32_t) * MLCAP * LTS <= sizeof(uint32_t) * 2 * NWORDS, "the staging area overlays the bitmaps");
static_assert(OWN_CAP <= 256, "mlist holds owner indices in a byte");
static_assert(STEP == 64 * 32 && STEP == 2 * ROW && (BUFB + STEP - 1) / STEP * 2 <= NWORDS / 32 + 1, "phase A writes both naw rows of its last step");

/* a scanned unit between its two halves: warp-uniform values, and one document per lane */
struct UnitRegs {
    uint32_t u, da, nd, extra, n_owners, n_ml, n_small /* tuples of the unit's small documents */; uint64_t total; bool needs_text;
    bool paged; /* more owning lines than OWN_CAP: the unit is scanned (and later written) one document at a time */
    bool long_line; /* an owner's line number exceeds the packed tuple's (ST_MAXLEN): the unit cannot take the deferred write */
    uint32_t dflag, dtot, dexcl, dlen; /* lane d < nd: document da + d */
};

struct WArgs {
    const uint8_t *bytes; const uint64_t *doc_off; uint32_t ndocs; uint64_t total_bytes;
    const uint32_t *tile_first; uint32_t ntiles;
    const uint64_t *ubase;                   /* [ntiles + 1] exclusive scan of units per tile */
    const WUnit *units;                      /* [units] descriptor of every unit (device: units are handed out one by one) */
    uint64_t *st_tuples, *st_blocks;         /* chain over the units' tuple counts (obm_warp.cuh: chain_publish / chain_resolve) */
    uint64_t units_max;                      /* capacity the chain arrays were carved for */
    const uint32_t *counts;                  /* tuple counts of large documents (k_large_resolve) */
    obm_tuple *out; uint64_t out_cap; uint64_t *tuple_off;
    uint32_t *status; unsigned long long *totals; uint32_t *ctl;
};
/* where a unit's text lies: computed ahead of the unit so that its bulk copy can be issued early.  doff: doc_off[da + lane]
 * on lanes 0..nd once the caller has loaded it with the prestaged copy (compute_unit loads it otherwise) */
struct UnitDesc { uint32_t u, da, db, extra, skew, span; uint64_t base_abs; bool valid; uint64_t doff; };
OBM_HD UnitDesc make_desc(const WArgs &A, uint32_t u, const WUnit &w) {
    const uint32_t nd = wu_nd(w);
    UnitDesc d{u, w.da, w.da + nd, wu_extra(w), 0, 0, 0, true, 0};
    if (nd) {
        const uint64_t abs0 = (uint64_t)(uintptr_t)A.bytes + w.off;
        d.base_abs = abs0 & ~15ull; d.skew = (uint32_t)(abs0 - d.base_abs); d.span = wu_span(w) + d.skew;
    }
    return d;
}
/* documents [da, db) of the batch as a unit: the same descriptor the set-up kernels write */
OBM_HD UnitDesc make_desc(const WArgs &A, uint32_t u, uint32_t da, uint32_t db, uint32_t extra) {
    return make_desc(A, u, pack_wunit(A.doc_off, da, db, extra));
}
OBM_HD uint32_t desc_load(const UnitDesc &d) { return (d.span + 15u) & ~15u; }
/* may the warp stage unit nxt's text (and load its document offsets) as soon as unit R is scanned?  Only when R's write
 * never reads the staged text again: R takes the deferred write, or the direct write of a unit without needs_text
 * (more than FIN_CAP tuples, long_line), which writes from the owner records and the staged marker tuples alone */
OBM_HD bool prestage_next(const UnitRegs &R, const UnitDesc &nxt) { return !R.needs_text && nxt.valid && nxt.db > nxt.da; }

struct WAcc { uint32_t markers, lexemes, exact, fatal; };
constexpr uint32_t MS_NONE = 0xFFFFFFFFu;

/* ---- bitmap helpers (phase B) ------------------------------------------------------------------------- */
OBM_HD bool w_is_nl(const UnitSet &S, uint32_t pos) { return (S.u.bm.nlw[pos >> 5] >> (pos & 31)) & 1u; }
OBM_HD bool w_is_sp(const UnitSet &S, uint32_t pos) { return (S.u.bm.spw[pos >> 5] >> (pos & 31)) & 1u; }
/* first position >= from whose special or newline bit is set, or hi */
OBM_FN uint32_t w_next_event(const UnitSet &S, uint32_t from, uint32_t hi) {
    if (from >= hi) return hi;
    uint32_t w = from >> 5;
    uint32_t m = (S.u.bm.spw[w] | S.u.bm.nlw[w]) & (0xFFFFFFFFu << (from & 31));
    const uint32_t wend = (hi + 31) >> 5;
    while (m == 0) {
        if (++w >= wend) return hi;
        m = S.u.bm.spw[w] | S.u.bm.nlw[w];
    }
    const uint32_t pos = w * 32 + OBMT_CTZ(m);
    return pos < hi ? pos : hi;
}
/* position after the last newline bit below pos (or lo) */
OBM_FN uint32_t w_line_start(const UnitSet &S, uint32_t pos, uint32_t lo) {
    uint32_t w = pos >> 5;
    uint32_t m = S.u.bm.nlw[w] & ((1u << (pos & 31)) - 1u);
    const uint32_t wlo = lo >> 5;
    while (m == 0) {
        if (w == wlo) return lo;
        m = S.u.bm.nlw[--w];
    }
#if defined(__CUDA_ARCH__)
    const uint32_t top = 31u - (uint32_t)__clz((int)m);
#else
    const uint32_t top = 31u - (uint32_t)__builtin_clz(m);
#endif
    const uint32_t ls = w * 32 + top + 1;
    return ls > lo ? ls : lo;
}
OBM_HD uint32_t w_nl_before(const WarpSmem &W, const UnitSet &S, uint32_t q) {
    const uint32_t w = q >> 5;
    static_assert(NWORDS % 2 == 0, "nlpre pairs the words");
    if (w >= NWORDS) return (uint32_t)W.nlpre[NWORDS / 2 - 1] + OBMT_POPC(S.u.bm.nlw[NWORDS - 2]) + OBMT_POPC(S.u.bm.nlw[NWORDS - 1]);
    return (uint32_t)W.nlpre[w >> 1] + ((w & 1u) ? OBMT_POPC(S.u.bm.nlw[w - 1]) : 0u) + OBMT_POPC(S.u.bm.nlw[w] & ((1u << (q & 31)) - 1u));
}

/* inclusive warp scan of a u32 */
#define OBMW_SCAN_INCL(v)                                                                                \
    do {                                                                                                 \
        _Pragma("unroll") for (uint32_t o_ = 1; o_ < 32; o_ <<= 1) { const uint32_t t_ = WSHFL_UP(v, o_); if (lane >= o_) v += t_; } \
    } while (0)

/* the line of owner record r, lexed by the generic ASCII lexer (hand-over target of the stepper): tuples into out[0..cap) */
template <class Src>
OBM_HD uint32_t generic_line(const obm::Tables &T, const Src &text, orec_t r, uint32_t dpos, uint32_t dend, obm_tuple *out, uint32_t cap,
                             uint32_t *mk, uint32_t *lx) {
    const uint32_t n = dend - dpos;
    uint32_t e = or_first(r); /* end of the line: the generic lexer's skipping is bounded by it (obmp::LineAccel) */
    while (e < n && text[dpos + e] != '\n') e++;
    const obmp::item_t it = obmp::make_marker_item(or_ls(r), or_first(r), or_line(r), 0, e);
    return obmp::k2_marker_item(T, obm::src_add(text, dpos), n, it, out, cap, mk, lx);
}

/* Go's utf8.DecodeRune validity over the bytes [q, e) of the staged text and no unicode.IsSpace code point beyond ASCII
 * (obm_tile.h utf8_plain explains why both): such a document keeps every line independent */
OBM_FN bool utf8_plain_w(const WarpSmem &W, uint32_t q, uint32_t e) {
    uint32_t p = q;
    while (p < e) {
        const uint32_t w = p >> 5;
        if (!((W.naw[w >> 5] >> (w & 31)) & 1u)) { p = (w + 1) << 5; continue; } /* all-ASCII word */
        const uint32_t wend = ((w + 1) << 5) < e ? ((w + 1) << 5) : e;
        while (p < wend) {
            const uint32_t b0 = W.text[p];
            if (b0 < 0x80) { p++; continue; }
            uint32_t need, lo = 0x80, hi = 0xBF;
            if (b0 >= 0xC2 && b0 <= 0xDF) need = 1;
            else if (b0 >= 0xE0 && b0 <= 0xEF) { need = 2; if (b0 == 0xE0) lo = 0xA0; if (b0 == 0xED) hi = 0x9F; }
            else if (b0 >= 0xF0 && b0 <= 0xF4) { need = 3; if (b0 == 0xF0) lo = 0x90; if (b0 == 0xF4) hi = 0x8F; }
            else return false;
            if (p + need >= e) return false; /* truncated at the end of the document */
            const uint32_t b1 = W.text[p + 1];
            if (b1 < lo || b1 > hi) return false;
            uint32_t b2 = 0;
            if (need >= 2) { b2 = W.text[p + 2]; if (b2 < 0x80 || b2 > 0xBF) return false; }
            if (need == 3) { const uint32_t b3 = W.text[p + 3]; if (b3 < 0x80 || b3 > 0xBF) return false; }
            if (b0 == 0xC2 && (b1 == 0x85 || b1 == 0xA0)) return false; /* Unicode white space */
            if (b0 == 0xE1 && b1 == 0x9A && b2 == 0x80) return false;
            if (b0 == 0xE2 && b1 == 0x80 && (b2 <= 0x8A || b2 == 0xA8 || b2 == 0xA9 || b2 == 0xAF)) return false;
            if (b0 == 0xE2 && b1 == 0x81 && b2 == 0x9F) return false;
            if (b0 == 0xE3 && b1 == 0x80 && b2 == 0x80) return false;
            p += need + 1;
        }
    }
    return true;
}

/* ---- phases A, B, C and the assembly of the tuple positions of documents [da, da + nd), whose text is staged at
 * [lo_pos, hi_pos) and whose starts / flags are in W.dstart[0..nd] / W.dflag[0..nd).  Returns false (nothing assembled)
 * when the range has more owning lines than OWN_CAP and the caller can split it (allow_page). ---- */
OBMW_DEV bool scan_range(WarpSmem &W, UnitSet &S, const WArgs &A, const obm::Tables &T, uint32_t u, uint32_t da, uint32_t nd,
                         uint32_t lo_pos, uint32_t hi_pos, bool allow_page, UnitRegs &R OBMW_PC_PARAM) {
    (void)A;
    const uint32_t lane = WLANE();
    uint32_t n_owners = 0, n_ml = 0;
    bool unstaged = false, long_line = false;
    if (nd) {
        const auto text = WTEXT(W);

        /* ---- A: steps of STEP bytes; lane L owns the 64 contiguous bytes [pos0, pos0 + 64) = bitmap words 2L, 2L+1 of the
         * step.  A lane whose bytes lie wholly at or past hi_pos neither loads nor stores: the last step can reach past
         * the staged text, the bitmaps and W.nlpre (nothing reads the words past hi_pos) ---- */
        const uint32_t s0 = lo_pos / STEP, s1 = (hi_pos + STEP - 1) / STEP;
        uint32_t nl_run = 0, own_run = 0, cin_step = 0, prev_top = 0, nextd = 1;
        for (uint32_t s = s0; s < s1; s++) {
            const uint32_t step0 = s * STEP, pos0 = step0 + lane * 64u;
            const bool live = pos0 < hi_pos;
            uint32_t xa[8] = {0, 0, 0, 0, 0, 0, 0, 0}, xb[8] = {0, 0, 0, 0, 0, 0, 0, 0};
            if (live) {
                const uint4 *q4 = reinterpret_cast<const uint4 *>(W.text + pos0);
                const uint4 a = q4[0], b = q4[1], c = q4[2], d = q4[3];
                xa[0] = a.x; xa[1] = a.y; xa[2] = a.z; xa[3] = a.w; xa[4] = b.x; xa[5] = b.y; xa[6] = b.z; xa[7] = b.w;
                xb[0] = c.x; xb[1] = c.y; xb[2] = c.z; xb[3] = c.w; xb[4] = d.x; xb[5] = d.y; xb[6] = d.z; xb[7] = d.w;
            }
            const uint64_t keep = range_mask64(pos0, lo_pos, hi_pos);
            Masks ma = classify32_t<false>(xa), mb = classify32_t<false>(xb);
            bool na0 = false, na1 = false; /* bytes >= 0x80 inside the range, per 32-byte word: their documents take the exact lexer */
            if (ma.hi | mb.hi) { /* rare; kept out of line (one copy of the exact classifier, one byte loop) to keep the hot loop small */
#pragma unroll 1
                for (uint32_t h = 0; h < 2; h++) { /* the carry-free byte test is only exact for 7-bit input */
                    uint32_t x[8];
#pragma unroll
                    for (int k = 0; k < 8; k++) x[k] = h ? xb[k] : xa[k];
                    Masks m = classify32_t<true>(x);
                    if (h) { m.hi = mb.hi; mb = m; } else { m.hi = ma.hi; ma = m; }
                }
                if (keep == ~0ull) { na0 = ma.hi != 0; na1 = mb.hi != 0; }
                else {
#pragma unroll 1
                    for (uint32_t k = 0; k < 64; k++) if (((keep >> k) & 1u) && W.text[pos0 + k] >= 0x80) { if (k < 32) na0 = true; else na1 = true; }
                }
            }
            uint64_t nl = ((uint64_t)ma.nl | ((uint64_t)mb.nl << 32)) & keep;
            const uint64_t hp = ((uint64_t)ma.hp | ((uint64_t)mb.hp << 32)) & keep, sl = ((uint64_t)ma.sl | ((uint64_t)mb.sl << 32)) & keep;
            const uint32_t nae = WBALLOT(na0), nao = WBALLOT(na1); /* even / odd words of the step */
            if (nae | nao) { /* rare: the two rows' W.naw entries interleave the ballots; exact attribution, byte by byte */
                const uint32_t w0 = spread16(nae) | (spread16(nao) << 1), w1 = spread16(nae >> 16) | (spread16(nao >> 16) << 1);
                if (lane == 0) { W.naw[2u * s] = w0; W.naw[2u * s + 1u] = w1; }
                if (lane < nd) {
                    const uint32_t q = W.dstart[lane], e = W.dstart[lane + 1];
                    for (uint32_t h = 0; h < 2; h++) {
                        for (uint32_t mm = h ? w1 : w0; mm; mm &= mm - 1) {
                            const uint32_t l0 = step0 + h * ROW + (OBMW_FFS(mm) - 1u) * 32u;
                            const uint32_t a = q > l0 ? q : l0, b = e < l0 + 32u ? e : l0 + 32u;
                            for (uint32_t p = a; p < b; p++) if (W.text[p] >= 0x80) W.dflag[lane] |= DF_NONASCII;
                        }
                    }
                }
            } else if (lane == 0) { W.naw[2u * s] = 0; W.naw[2u * s + 1u] = 0; }
            /* "//": a '/' whose successor is a '/' (the successor of the lane's last byte sits in the next lane's bytes) */
            const uint64_t nxt = (pos0 + 64u < hi_pos && W.text[pos0 + 64u] == '/') ? (1ull << 63) : 0ull;
            uint64_t ss = sl & ((sl >> 1) | nxt);
            /* virtual newline on the byte before every document start (a line starts there, whatever the byte is) */
            while (nextd < nd) {
                const uint32_t q = W.dstart[nextd];
                if (q > lo_pos) {
                    if (q - 1u >= step0 + STEP) break;
                    if (((q - 1u - step0) >> 6) == lane) { const uint64_t bit = 1ull << ((q - 1u) & 63u); nl |= bit; ss &= ~bit; }
                }
                nextd++;
            }
            const uint64_t sp = hp | ss;
            const uint64_t ev = nl | sp;
            /* line starts: after every newline, and at the first byte of the range */
            const uint32_t top = (uint32_t)(nl >> 63);
            uint32_t up = WSHFL_UP(top, 1);
            if (lane == 0) up = prev_top;
            uint64_t M = (nl << 1) | up;
            if (s == s0 && lo_pos < hi_pos && ((lo_pos - step0) >> 6) == lane) M |= 1ull << (lo_pos & 63u);
            /* first event of every line: (~ev + M) & ev, the carry resolved across lanes by generate / propagate */
            const uint64_t nev = ~ev, sum = nev + M;
            const bool G = sum < nev; /* carry out of the lane's 64 bits */
            const uint32_t Gb = WBALLOT(G), Pb = WBALLOT(ev == 0 && !G);
            uint32_t cout;
            const uint32_t Cm = obmt::carry_lookahead32(Gb, Pb, cin_step, &cout);
            const uint32_t cin = (Cm >> lane) & 1u;
            uint64_t own = (sum + cin) & ev & sp;
            cin_step = cout;
            prev_top = WSHFL(top, 31);
            const uint32_t wi = 2u * (s * 32u + lane);
            if (live) {
                S.u.bm.nlw[wi] = (uint32_t)nl; S.u.bm.nlw[wi + 1u] = (uint32_t)(nl >> 32);
                S.u.bm.spw[wi] = (uint32_t)sp; S.u.bm.spw[wi + 1u] = (uint32_t)(sp >> 32);
            }
            uint32_t cnt = OBMW_POPC64(nl) | (OBMW_POPC64(own) << 16); /* a step holds at most 2,048 of either */
            const uint32_t mine = cnt;
            OBMW_SCAN_INCL(cnt);
            const uint32_t excl = cnt - mine;
            if (live) W.nlpre[s * 32u + lane] = (uint16_t)(nl_run + (excl & 0xFFFFu));
            uint32_t o = own_run + (excl >> 16);
            while (own) {
                if (o < OWN_CAP) S.orec[o] = pos0 + (OBMW_FFS64(own) - 1u);
                o++; own &= own - 1u;
            }
            const uint32_t tot = WSHFL(cnt, 31);
            nl_run += tot & 0xFFFFu; own_run += tot >> 16;
        }
        WSYNC();
        n_owners = own_run;
        if (n_owners > OWN_CAP) {
            if (allow_page) return false;
            n_owners = 0; if (lane < nd) W.dflag[lane] |= DF_QOVERFLOW;
        }
        if (lane < nd && W.dflag[lane] == DF_NONASCII && utf8_plain_w(W, W.dstart[lane], W.dstart[lane + 1])) W.dflag[lane] = DF_UNI;
        WSYNC();
        OBMW_PC_MARK(PC_A);

        /* ---- B: owners ---- */
        for (uint32_t o0 = 0; o0 < n_owners; o0 += 32) {
            const uint32_t o = o0 + lane; const bool valid = o < n_owners;
            bool marker = false;
            if (valid) {
                const uint32_t first = (uint32_t)S.orec[o];
                const uint32_t ls = w_line_start(S, first, lo_pos);
                uint32_t dlo = 0, dhi = nd; /* last d with dstart[d] <= ls */
                while (dhi - dlo > 1) { const uint32_t mid = (dlo + dhi) >> 1; if (W.dstart[mid] <= ls) dlo = mid; else dhi = mid; }
                const uint32_t d = dlo, dpos = W.dstart[d];
                const uint32_t df = W.dflag[d];
                bool uni = false;
                if (df & DF_UNI) { /* does the line hold bytes >= 0x80?  Only marker lines care:
                                    * lex / lexComment (state.go:15-57) look for '#', "//", '+' and '\n' and nothing else */
                    const uint32_t dend = W.dstart[d + 1];
                    uint32_t e = first;
                    for (;;) { if (e >= dend) { e = dend; break; } if (w_is_nl(S, e) && text[e] == '\n') break; e = w_next_event(S, e + 1, hi_pos); }
                    const uint32_t last = e < hi_pos ? e : hi_pos - 1u;
                    for (uint32_t w = ls >> 5; w <= (last >> 5); w++) uni |= ((W.naw[w >> 5] >> (w & 31)) & 1u) != 0;
                    if (uni) { uni = false; for (uint32_t q = ls; q <= last; q++) uni |= W.text[q] >= 0x80; } /* the words are shared with the neighbouring lines */
                }
                if (df & DF_EXACT) { S.orec[o] = make_orec(ls - dpos, first - dpos, 0, false, false, true, d, 0); S.opos[o] = 0; }
                else {
                    const uint32_t line = 1 + w_nl_before(W, S, ls) - w_nl_before(W, S, dpos);
                    long_line |= line > ST_MAXLEN;
                    const uint32_t c = text[first];
                    uint32_t plus = first;
                    marker = c == '+';
                    if (!marker) { /* is there a '+' further on this line?  (state.go:46-57: lexComment looks for nothing else) */
                        uint32_t e = first;
                        for (;;) {
                            if (w_is_nl(S, e)) break; /* a special on the document's last byte */
                            e = w_next_event(S, e + 1, hi_pos);
                            if (e >= hi_pos || !w_is_sp(S, e)) break;
                            if (text[e] == '+') { marker = true; plus = e; break; }
                        }
                    }
                    const uint32_t pd = plus - first < PD_GENERIC ? plus - first : PD_GENERIC;
                    if (marker && uni) WATOMIC_OR(&W.dflag[d], DF_INTERACT); /* names, values and the letter after '+' are judged by Unicode classes: the exact lexer's */
                    S.orec[o] = make_orec(ls - dpos, first - dpos, line, marker, c == '/', false, d, pd);
                    if (!marker) S.opos[o] = (uint16_t)(line == 1 ? 1u : 2u);
                }
            }
            const uint32_t bal = WBALLOT(marker);
            if (marker) S.mlist[n_ml + OBMT_POPC(bal & ((1u << lane) - 1u))] = (uint8_t)o;
            n_ml += OBMT_POPC(bal);
        }
        WSYNC(); /* the bitmaps are dead from here on: their space becomes the staging area */

        if (lane < nd) W.dflag[lane] &= ~DF_UNI; /* from here on a set flag means: the exact lexer */
        WSYNC();
        OBMW_PC_MARK(PC_B);
        /* ---- C: marker lines, a lane per line; the first MLCAP lines stage their tuples ---- */
        for (uint32_t k0 = 0; k0 < n_ml; k0 += 32) {
            const uint32_t k = k0 + lane; const bool on = k < n_ml;
            if (on) {
                const uint32_t o = S.mlist[k];
                const orec_t r = S.orec[o];
                const uint32_t d = or_doc(r), dpos = W.dstart[d], dend = W.dstart[d + 1];
                const bool staged = k0 == 0;
                PackSink sink(S.u.c.stage + lane * LTS, staged ? LTS : 0u);
                uint32_t res = FL_FALLBACK;
                if (or_plusd(r) != PD_GENERIC)
                    res = fast_line(text, dpos + or_first(r), dpos + or_first(r) + or_plusd(r), dpos + or_ls(r), or_line(r), dpos, dend, sink);
                uint32_t cntv; bool stg = staged;
                if (res == FL_OK) { cntv = sink.n; if (sink.ovf) stg = false; OBMW_STAT(fast); }
                else { /* outside the well-formed grammar: the generic lexer decides (count only; written in place later) */
                    OBMW_STAT(generic);
                    const uint32_t gr = generic_line(T, text, r, dpos, dend, nullptr, 0, nullptr, nullptr);
                    S.orec[o] = r | ((orec_t)PD_GENERIC << 50); /* remember: this line is the generic lexer's */
                    cntv = obmp::mres_tuples(gr);
                    if (obmp::mres_irregular(gr)) WATOMIC_OR(&W.dflag[d], DF_INTERACT);
                    stg = false;
                }
                if (cntv >= 0xFFFFu) { WATOMIC_OR(&W.dflag[d], DF_INTERACT); cntv = 0; }
                S.opos[o] = (uint16_t)cntv;
                if (staged) S.u.c.mstat[lane] = (stg && cntv) ? (sink.mk | (sink.lx << 8) | (cntv << 16)) : MS_NONE; /* cntv <= LTS: the counters fit */
                if (cntv && !stg) unstaged = true;
            }
        }
        WSYNC();
        OBMW_PC_MARK(PC_C);
    }

    /* ---- assembly: counts -> positions inside the unit ---- */
    uint32_t dflag = 0, dtot = 0, dlen = 0;
    if (lane < nd) {
        dflag = W.dflag[lane];
        const uint32_t dpos = W.dstart[lane], dend = W.dstart[lane + 1];
        dlen = dend - dpos;
        if (dflag) { /* documents that need the exact lexer (as in r01's K2) */
            obm::SmallSink sink(nullptr, 0);
            obmp::doc_exact(T, W.text + dpos, dlen, sink);
            dtot = sink.n_tuples;
        }
        /* first owner of the document: owners are in position order, hence grouped by document */
        uint32_t lo = 0, hi = n_owners;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (or_doc(S.orec[mid]) < lane) lo = mid + 1; else hi = mid; }
        W.dfo[lane] = (uint16_t)lo;
    }
    if (lane == nd) W.dfo[nd] = (uint16_t)n_owners;
    WSYNC();
    /* exclusive prefix over the owners' tuple counts (owners of flagged documents count 0) */
    uint32_t run = 0;
    for (uint32_t o0 = 0; o0 < n_owners; o0 += 32) {
        const uint32_t o = o0 + lane;
        uint32_t c = 0;
        if (o < n_owners) { c = S.opos[o]; if (W.dflag[or_doc(S.orec[o])]) c = 0; }
        uint32_t v = c;
        OBMW_SCAN_INCL(v);
        if (o < n_owners) S.opos[o] = (uint16_t)(run + v - c);
        run += WSHFL(v, 31);
    }
    WSYNC();
    uint32_t p0 = 0; /* prefix of the document's first owner */
    if (lane < nd) {
        const uint32_t f0 = W.dfo[lane], f1 = W.dfo[lane + 1];
        p0 = f0 < n_owners ? S.opos[f0] : run;
        const uint32_t p1 = f1 < n_owners ? S.opos[f1] : run;
        if (!dflag) dtot = p1 - p0 + 1u; /* + EOF */
    }
    uint32_t dincl = lane < nd ? dtot : 0u;
    OBMW_SCAN_INCL(dincl);
    const uint32_t dexcl = dincl - (lane < nd ? dtot : 0u);
    uint64_t total = WSHFL(dincl, 31);
    if (lane < nd) W.dcnt[lane] = (uint16_t)(dexcl - p0); /* owner prefix + this = tuple position inside the unit */
    WSYNC();
    for (uint32_t o0 = 0; o0 < n_owners; o0 += 32) {
        const uint32_t o = o0 + lane;
        if (o < n_owners) S.opos[o] = (uint16_t)(W.dcnt[or_doc(S.orec[o])] + S.opos[o]);
    }
    WSYNC();
    R.n_small = (uint32_t)total;
    R.u = u; R.da = da; R.nd = nd; R.extra = 0; R.n_owners = n_owners; R.n_ml = n_ml; R.total = total;
    R.dflag = dflag; R.dtot = dtot; R.dexcl = dexcl; R.dlen = dlen;
    R.needs_text = WBALLOT(unstaged || dflag != 0) != 0;
    R.paged = false;
    R.long_line = WBALLOT(long_line) != 0;
    OBMW_PC_MARK(PC_ASM);
    return true;
}

/* ---- first half of a unit: stage its text, scan it, assemble the tuple positions.  prestaged: the caller has issued the
 * text's bulk copy and, with it, loaded D.doff ---- */
template <class Hooks>
OBMW_DEV void compute_unit(WarpSmem &W, UnitSet &S, const WArgs &A, const obm::Tables &T, Hooks &H, const UnitDesc &D, bool prestaged, UnitRegs &R OBMW_PC_PARAM) {
    const uint32_t lane = WLANE();
    const uint32_t u = D.u, da = D.da, nd = D.db - D.da, extra = D.extra;
    uint32_t lo_pos = 0, hi_pos = 0;
    if (nd) {
        const uint32_t skew = D.skew, span = D.span, load = desc_load(D);
        const uint64_t b0 = (D.base_abs + skew) - (uint64_t)(uintptr_t)A.bytes;
        lo_pos = skew; hi_pos = span;
        uint64_t doff = D.doff;
        if (!prestaged) { H.stage(W, (const void *)(uintptr_t)D.base_abs, load); if (lane <= nd) doff = A.doc_off[da + lane]; }
        if (lane <= nd) W.dstart[lane] = (uint32_t)(doff - b0) + skew;
        if (lane < nd) W.dflag[lane] = 0;
        WSYNC();
        H.stage_wait(W, load);
        OBMW_PC_MARK(PC_STAGE);
    }
    /* one scan of the whole range; when it has more owning lines than the owner table holds (lines of a few bytes) the
     * same call site then counts it document by document (write_unit scans each document again when it writes it) */
    uint32_t mypos = 0, my_tot = 0, my_flag = 0;
    for (uint32_t j = 0xFFFFFFFFu;;) {
        const bool whole = j == 0xFFFFFFFFu;
        uint32_t pj = lo_pos, ej = hi_pos;
        if (!whole) {
            pj = WSHFL(mypos, j); ej = WSHFL(mypos, j + 1);
            if (lane == 0) { W.dstart[0] = pj; W.dstart[1] = ej; W.dflag[0] = 0; }
            WSYNC();
        }
        const bool ok = scan_range(W, S, A, T, u, whole ? da : da + j, whole ? nd : 1u, pj, ej, whole && nd > 1, R OBMW_PC_ARG);
        if (whole) {
            if (ok) break;
            mypos = lane <= nd ? W.dstart[lane] : 0u;
            WSYNC();
            j = 0;
            continue;
        }
        const uint32_t tj = WSHFL(R.dtot, 0), fj = WSHFL(R.dflag, 0);
        if (lane == j) { my_tot = tj; my_flag = fj; }
        WSYNC();
        if (++j < nd) continue;
        if (lane <= nd) W.dstart[lane] = mypos;
        if (lane < nd) W.dflag[lane] = my_flag;
        WSYNC();
        uint32_t dincl = lane < nd ? my_tot : 0u;
        OBMW_SCAN_INCL(dincl);
        const uint32_t nextpos = WSHFL(mypos, (lane + 1) & 31u);
        R.u = u; R.da = da; R.nd = nd; R.n_owners = 0; R.n_ml = 0;
        R.dflag = my_flag; R.dtot = my_tot; R.dexcl = dincl - (lane < nd ? my_tot : 0u);
        R.dlen = lane < nd ? nextpos - mypos : 0u;
        R.total = WSHFL(dincl, 31); R.n_small = (uint32_t)R.total;
        R.needs_text = true; R.paged = true;
        break;
    }
    R.extra = extra;
    if (extra) R.total += A.counts[da + nd];
}

/* staged marker tuples: staged line k (lane k < ns) holds c tuples whose place is [rel, rel + c) inside the unit;
 * put(position, packed tuple) stores one.  A line per round, a lane per tuple */
template <class Put>
OBMW_DEV void copy_staged(const UnitSet &S, uint32_t ns, uint32_t c, uint32_t rel, Put put) {
    const uint32_t lane = WLANE();
    for (uint32_t k = 0; k < ns; k++) {
        const uint32_t ck = WSHFL(c, k), rk = WSHFL(rel, k);
        if (lane < ck) put(rk + lane, S.u.c.stage[k * LTS + lane]);
    }
}

/* ---- deferred path: the unit's tuples packed into W.fin in final order (only units without needs_text) -------
 * Returns false when the unit does not fit (more than FIN_CAP tuples, a line number beyond the packed form): the
 * caller then writes it directly (write_unit). */
OBMW_DEV bool assemble_fin(WarpSmem &W, UnitSet &S, const UnitRegs &R, WAcc &acc) {
    const uint32_t lane = WLANE();
    const uint32_t nd = R.nd, n_owners = R.n_owners, n_ml = R.n_ml;
    if (R.n_small > FIN_CAP || R.long_line) return false;
    if (lane < nd) { W.fin[R.dexcl + R.dtot - 1u] = st_pack(OBM_K_EOF, R.dlen, 0); acc.lexemes++; }
    for (uint32_t o0 = 0; o0 < n_owners; o0 += 32) {
        const uint32_t o = o0 + lane;
        if (o >= n_owners) continue;
        const orec_t r = S.orec[o];
        if (or_dead(r) || or_marker(r)) continue;
        uint32_t at = S.opos[o];
        if (or_line(r) != 1) W.fin[at++] = st_pack(OBM_K_LINE, or_ls(r), or_line(r));
        W.fin[at] = st_pack(OBM_K_COMMENT, or_first(r), or_slash2(r) ? 2 : 1);
        acc.lexemes++;
    }
    {
        const uint32_t ns = n_ml < MLCAP ? n_ml : MLCAP;
        uint32_t c = 0, rel = 0;
        if (lane < ns) {
            const uint32_t ms = S.u.c.mstat[lane]; /* never MS_NONE here: every marker line with tuples is staged */
            if (ms != MS_NONE) { c = ms >> 16; rel = S.opos[S.mlist[lane]]; acc.markers += ms & 0xFFu; acc.lexemes += (ms >> 8) & 0xFFu; }
        }
        copy_staged(S, ns, c, rel, [&](uint32_t at, uint32_t v) { W.fin[at] = v; });
    }
    WSYNC();
    return true;
}
OBMW_DEV void write_fin(const WarpSmem &W, const WArgs &A, const UnitRegs &R, uint32_t nunits, uint64_t base) {
    const uint32_t lane = WLANE();
    if (lane == 0) {
        if (R.u == 0) A.tuple_off[0] = 0;
        if (R.u == nunits - 1 && A.out && base + R.total > A.out_cap) A.status[0] = 1;
        if (R.extra) A.tuple_off[R.da + R.nd + 1] = base + R.total;
    }
    if (lane < R.nd) A.tuple_off[R.da + lane + 1] = base + R.dexcl + R.dtot;
    if (A.out != nullptr && A.out_cap != 0) {
        obm_tuple *dst = A.out + base;
        if (base + R.n_small <= A.out_cap) for (uint32_t f = lane; f < R.n_small; f += 32) dst[f] = st_unpack(W.fin[f]);
        else for (uint32_t f = lane; f < R.n_small; f += 32) if (base + f < A.out_cap) dst[f] = st_unpack(W.fin[f]);
    }
    WSYNC(); /* fin is free again */
}

/* ---- second half: the unit's tuples at their final positions (base = tuples of all earlier units) ----------
 * The direct path: units with needs_text, or too large for W.fin; written before the warp stages its next unit. */
OBMW_DEV void write_range(WarpSmem &W, UnitSet &S, const WArgs &A, const obm::Tables &T, const UnitRegs &R, uint64_t base, WAcc &acc);
OBMW_DEV void write_unit(WarpSmem &W, UnitSet &S, const WArgs &A, const obm::Tables &T, const UnitRegs &R, uint32_t nunits, uint64_t base, WAcc &acc
                         OBMW_PC_PARAM) {
    const uint32_t lane = WLANE();
    if (lane == 0) {
        if (R.u == 0) A.tuple_off[0] = 0;
        if (R.u == nunits - 1 && A.out && base + R.total > A.out_cap) A.status[0] = 1;
        if (R.extra) A.tuple_off[R.da + R.nd + 1] = base + R.total;
    }
    /* a paged unit: every document is scanned again, alone, and written at its place (same call site as the usual case) */
    const uint32_t mypos = (R.paged && lane <= R.nd) ? W.dstart[lane] : 0u;
    if (R.paged) WSYNC();
    const uint32_t npages = R.paged ? R.nd : 1u;
    for (uint32_t j = 0; j < npages; j++) {
        UnitRegs Rj = R;
        uint64_t bj = base;
        if (R.paged) {
            const uint32_t pj = WSHFL(mypos, j), ej = WSHFL(mypos, j + 1);
            bj = base + WSHFL(R.dexcl, j);
            if (lane == 0) { W.dstart[0] = pj; W.dstart[1] = ej; W.dflag[0] = 0; }
            WSYNC();
            scan_range(W, S, A, T, R.u, R.da + j, 1, pj, ej, false, Rj OBMW_PC_ARG);
        }
        write_range(W, S, A, T, Rj, bj, acc);
        OBMW_PC_MARK(PC_WRITE);
    }
}
/* the documents of a scanned range: tuples at their final positions (base = tuples before the range's first document) */
OBMW_DEV void write_range(WarpSmem &W, UnitSet &S, const WArgs &A, const obm::Tables &T, const UnitRegs &R, uint64_t base, WAcc &acc) {
    const uint32_t lane = WLANE();
    const uint32_t nd = R.nd, n_owners = R.n_owners, n_ml = R.n_ml;
    const bool writing = A.out != nullptr && A.out_cap != 0;
    if (nd == 0) return;
    if (lane < nd) {
        const uint64_t at = base + R.dexcl;
        A.tuple_off[R.da + lane + 1] = at + R.dtot;
        if (R.dflag) { /* only with needs_text: the text and the document table are still this unit's */
            acc.exact++;
            if (writing) {
                const uint64_t roomv = at < A.out_cap ? A.out_cap - at : 0;
                obm::SmallSink sink(A.out + at, roomv > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)roomv);
                const int st = obmp::doc_exact(T, W.text + W.dstart[lane], R.dlen, sink);
                acc.markers += sink.n_markers; acc.lexemes += sink.n_lexemes; acc.fatal += (st == obm::RUN_FATAL) ? 1u : 0u;
            }
        } else {
            const uint64_t eof_at = at + R.dtot - 1u;
            if (writing && eof_at < A.out_cap) A.out[eof_at] = OBM_TUPLE(OBM_K_EOF, R.dlen, 0);
            acc.lexemes++;
        }
    }
    /* plain lines in place */
    for (uint32_t o0 = 0; o0 < n_owners; o0 += 32) {
        const uint32_t o = o0 + lane;
        if (o >= n_owners) continue;
        const orec_t r = S.orec[o];
        if (or_dead(r) || or_marker(r)) continue;
        if (R.needs_text && W.dflag[or_doc(r)]) continue; /* without needs_text no document is flagged */
        const uint64_t at = base + S.opos[o];
        if (writing) {
            uint32_t k = 0;
            if (or_line(r) != 1) { if (at < A.out_cap) A.out[at] = OBM_TUPLE(OBM_K_LINE, or_ls(r), or_line(r)); k = 1; }
            if (at + k < A.out_cap) A.out[at + k] = OBM_TUPLE(OBM_K_COMMENT, or_first(r), or_slash2(r) ? 2 : 1);
        }
        acc.lexemes++;
    }
    /* marker lines that are not staged are lexed again, straight to their place (needs_text) */
    if (R.needs_text) {
        const auto text = WTEXT(W);
        for (uint32_t k0 = 0; k0 < n_ml; k0 += 32) {
            const uint32_t k = k0 + lane;
            if (k >= n_ml) continue;
            if (k0 == 0 && S.u.c.mstat[lane] != MS_NONE) continue; /* staged */
            const uint32_t o = S.mlist[k];
            const orec_t r = S.orec[o];
            const uint32_t d = or_doc(r), dpos = W.dstart[d], dend = W.dstart[d + 1];
            if (W.dflag[d] || !writing) continue;
            const uint64_t at = base + S.opos[o];
            const uint64_t roomv = at < A.out_cap ? A.out_cap - at : 0;
            const uint32_t rc = roomv > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)roomv;
            if (or_plusd(r) != PD_GENERIC) {
                DirectSink sink(A.out + at, rc);
                fast_line(text, dpos + or_first(r), dpos + or_first(r) + or_plusd(r), dpos + or_ls(r), or_line(r), dpos, dend, sink);
                acc.markers += sink.mk; acc.lexemes += sink.lx;
            } else {
                uint32_t mk = 0, lx = 0;
                generic_line(T, text, r, dpos, dend, A.out + at, rc, &mk, &lx);
                acc.markers += mk; acc.lexemes += lx;
            }
        }
    }
    /* staged marker tuples (a line's tuples are contiguous on both sides) */
    {
        const uint32_t ns = n_ml < MLCAP ? n_ml : MLCAP;
        uint32_t c = 0, rel = 0;
        if (lane < ns) {
            const uint32_t ms = S.u.c.mstat[lane];
            const uint32_t o = S.mlist[lane];
            if (ms != MS_NONE && !(R.needs_text && W.dflag[or_doc(S.orec[o])])) {
                c = ms >> 16; rel = S.opos[o];
                acc.markers += ms & 0xFFu; acc.lexemes += (ms >> 8) & 0xFFu;
            }
        }
        if (writing) copy_staged(S, ns, c, rel, [&](uint32_t f, uint32_t v) { if (base + f < A.out_cap) A.out[base + f] = st_unpack(v); });
    }
    WSYNC();
}

} /* namespace obmw */
#endif
