/*
 * hostsim.cpp -- TEST INFRASTRUCTURE.  Compiles the product's lexer core (obm_core.h, the same
 * source the CUDA kernels instantiate) for the host so that `pytest -m "not gpu"` can check the
 * tuple stream + decoder logic against the oracle without a GPU.  Never loaded by the product
 * package; libobmarkers.so has no host lexing entry point.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include "../../operator-builder_b200/csrc/go_unicode_tables.h"
#include "../../operator-builder_b200/csrc/obm_core.h"

static const char F64[] = GO_F64_OVERFLOW_DIGITS;
static const obm::Tables TBL = { GO_LETTER_RANGES, GO_LETTER_RANGES_N, GO_NUMBER_RANGES, GO_NUMBER_RANGES_N, F64 };

extern "C" {
/* whole-document exact path; returns the tuple count (writes at most cap) */
uint64_t hs_lex_doc(const uint8_t *doc, uint32_t n, obm_tuple *out, uint64_t cap, uint32_t *n_markers, uint32_t *n_lexemes) {
    obm::WriteSink sink(out, cap);
    obm::Lexer<obm::WriteSink> lx(TBL, doc, n, sink);
    lx.run<false>();
    if (n_markers) *n_markers = sink.n_markers;
    if (n_lexemes) *n_lexemes = sink.n_lexemes;
    return sink.n_tuples;
}
/* per-line composition, the way the fast kernel assembles a document: one LINE_MODE lexer per
 * physical line that has not been swallowed by an earlier owner, EOF appended unless fatal. */
uint64_t hs_lex_doc_by_lines(const uint8_t *doc, uint32_t n, obm_tuple *out, uint64_t cap) {
    obm::WriteSink sink(out, cap);
    uint32_t pos = 0, line = 1;
    bool fatal = false;
    while (pos < n) {
        obm::Lexer<obm::WriteSink> lx(TBL, doc, n, sink, pos, line, pos, !(line == 1 && pos == 0));
        int st = lx.run<true>();
        if (st == obm::RUN_FATAL) { fatal = true; break; }
        if (st == obm::RUN_EOF) break;
        pos = lx.p; line = lx.line_p;
    }
    if (!fatal) sink.put(OBM_K_EOF, n, 0);
    return sink.n_tuples;
}
int hs_parse_float_err(const uint8_t *s, uint32_t n) { return obm::parse_float_err(TBL, s, n); }
int hs_atoi_err(const uint8_t *s, uint32_t n) { return obm::atoi_err(s, n); }
}

/* ---------------------------------------------------------------------------------------------
 * Unicode hooks (tests/test_unicode13.py): the product's classes and quoter over the host tables, and
 * batch lex + decode in the record format of the oracle's obo_lex_batch, so that millions of one-line
 * documents compare as one byte string.
 * ------------------------------------------------------------------------------------------- */
#include <string>
#include <vector>
#include "../../include/obmarkers.h"
#include "../../operator-builder_b200/csrc/obm_quote.h"

namespace {
/* obm_decode_doc of one document appended to `out` -> its lexeme count */
int64_t decode_append(std::string &out, const uint8_t *doc, uint64_t n, const obm_tuple *t, uint64_t nt) {
    uint8_t *p = nullptr; uint64_t len = 0;
    int64_t c = obm_decode_doc(doc, n, t, nt, &p, &len);
    if (c < 0) return c;
    out.append((const char *)p, len);
    free(p);
    return c;
}
/* the serialised batch handed to the caller (release with obm_free) */
int finish(const std::string &buf, uint8_t **out, uint64_t *out_len) {
    uint8_t *p = (uint8_t *)malloc(buf.size() ? buf.size() : 1);
    if (!p) return OBM_E_NOMEM;
    memcpy(p, buf.data(), buf.size());
    *out = p; *out_len = buf.size();
    return 0;
}
} // namespace

extern "C" {
/* out[i] bit 0: obm::is_letter, bit 1: obm::is_number, bit 2: obm::is_space, bit 3: obm::go_is_print (strconv.IsPrint) */
void hs_classify(const int32_t *cps, uint64_t n, uint8_t *out) {
    for (uint64_t i = 0; i < n; i++) {
        const int r = cps[i];
        out[i] = (uint8_t)(obm::is_letter(TBL, r) | obm::is_number(TBL, r) << 1 | obm::is_space(r) << 2 | obm::go_is_print(r) << 3);
    }
}
/* strconv.Quote of s as the decoder and the parser print it; returns the full length (writes at most cap) */
uint64_t hs_go_quote(const uint8_t *s, uint64_t n, uint8_t *out, uint64_t cap) {
    const std::string q = obm::go_quote(std::string((const char *)s, n));
    memcpy(out, q.data(), q.size() < cap ? q.size() : cap);
    return q.size();
}
/* every document through the host build of the exact lexer, then obm_decode_doc: stream_off[ndocs+1] and n_lexemes[ndocs]
 * as obo_lex_batch fills them */
int hs_lex_decode_batch(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, uint8_t **out, uint64_t *out_len,
                        uint64_t *stream_off, uint64_t *n_lexemes) {
    std::string buf;
    std::vector<obm_tuple> t;
    for (uint32_t d = 0; d < ndocs; d++) {
        const uint8_t *doc = bytes + doc_off[d];
        const uint32_t n = (uint32_t)(doc_off[d + 1] - doc_off[d]);
        uint64_t nt = 2 * (uint64_t)n + 16;
        for (;;) {
            t.resize(nt);
            const uint64_t got = hs_lex_doc(doc, n, t.data(), nt, nullptr, nullptr);
            if (got <= nt) { nt = got; break; }
            nt = got;
        }
        stream_off[d] = buf.size();
        const int64_t c = decode_append(buf, doc, n, t.data(), nt);
        if (c < 0) return (int)c;
        n_lexemes[d] = (uint64_t)c;
    }
    stream_off[ndocs] = buf.size();
    return finish(buf, out, out_len);
}
/* obm_decode_doc over given tuples: document d's are tuples[tuple_off[d] .. tuple_off[d+1]) */
int hs_decode_batch(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, const obm_tuple *tuples, const uint64_t *tuple_off,
                    uint8_t **out, uint64_t *out_len, uint64_t *stream_off) {
    std::string buf;
    for (uint32_t d = 0; d < ndocs; d++) {
        stream_off[d] = buf.size();
        const int64_t c = decode_append(buf, bytes + doc_off[d], doc_off[d + 1] - doc_off[d], tuples + tuple_off[d], tuple_off[d + 1] - tuple_off[d]);
        if (c < 0) return (int)c;
    }
    stream_off[ndocs] = buf.size();
    return finish(buf, out, out_len);
}
}

/* ---------------------------------------------------------------------------------------------
 * CTA emulation of the tile fast path (obm_fast.cuh's k_tile_scan): the same phase functions from
 * obm_tile.h, run for tid = 0..NT-1 between "barriers", tiles visited in order (which is what the
 * look-back chain enforces on the device).
 * ------------------------------------------------------------------------------------------- */
#include <vector>
#include "../../operator-builder_b200/csrc/obm_tile.h"
#include "../../operator-builder_b200/csrc/obm_pipe.h"

namespace {
using obmt::Smem;

struct Emu {
    Smem S;
    uint32_t sub_total = 0;
    bool uni_lines = false; /* the two-stage pipeline lexes lines with non-ASCII bytes one by one (doc_prep) */
    uint64_t total_bytes = 0; /* size of the packed batch (bytes after a sub-batch that the bulk copy also brings in) */
    /* P1..P4: stage, classify, doc prep, bit-parallel line scan -> S.owner[] = first special of each owning line */
    uint32_t scan(const uint8_t *bytes, const uint64_t *doc_off, uint32_t da, uint32_t db, uint32_t fake_skew) {
        const uint32_t nd = db - da;
        const uint64_t b0 = doc_off[da], b1 = doc_off[db];
        (void)fake_skew; /* callers place the batch at the alignment they want to test (tests/hostsim/__init__.py) */
        const uint32_t skew = (uint32_t)((uintptr_t)(bytes + b0) & 15u); /* as on the device: from the absolute address, so that
                                                                          * K1's 32-byte words and K2's aligned 4-byte loads line up */
        const uint32_t span = (uint32_t)(b1 - b0) + skew;
        S.nd = nd; S.lo_pos = skew; S.hi_pos = span; S.n_owners = 0;
        memset(S.data, 0x2B, sizeof S.data); /* '+' garbage outside the loaded range must never matter */
        memcpy(S.data + skew, bytes + b0, (size_t)(b1 - b0));
        /* the device's bulk copy starts at the 16-byte boundary below the first document and ends at the one above the
         * last: the neighbouring documents' real bytes are in the buffer too (they decide, e.g., whether the 32-byte
         * word around a document boundary counts as non-ASCII).  `total` bounds what exists after the batch. */
        if (b0 >= skew) memcpy(S.data, bytes + b0 - skew, skew);
        {
            const uint32_t load = (span + 15u) & ~15u;
            const uint64_t avail = total_bytes > b1 ? total_bytes - b1 : 0;
            const uint32_t extra = load - span < avail ? load - span : (uint32_t)avail;
            if (extra) memcpy(S.data + span, bytes + b1, extra);
        }
        for (uint32_t t = 0; t <= nd; t++) S.dstart[t] = (uint32_t)(doc_off[da + t] - b0) + skew;
        const uint32_t nwords = (span + 31) >> 5;
        for (uint32_t wi = 0; wi < obmt::NW; wi++) {
            if (wi < ((nwords + 31u) & ~31u)) obmt::classify_word(S, wi); else { S.nlw[wi] = 0; S.spw[wi] = 0; }
        }
        for (uint32_t t = 0; t < nd; t++) obmt::doc_prep(S, t, uni_lines);
        /* P4: per-thread generate/propagate, warp look-ahead from emulated ballots, cross-warp resolve */
        std::vector<uint32_t> my_nl(obmt::NT), my_own(obmt::NT), g(obmt::NT), pr(obmt::NT), cin_t(obmt::NT);
        std::vector<obmt::LineBits> lbs(obmt::NT);
        auto load = [&](uint32_t t, uint32_t (&nl)[obmt::WPT], uint32_t (&sp)[obmt::WPT], uint32_t (&lm)[obmt::WPT]) {
            for (uint32_t j = 0; j < obmt::WPT; j++) { nl[j] = S.nlw[t * obmt::WPT + j]; sp[j] = S.spw[t * obmt::WPT + j]; }
            obmt::line_starts(S, t, nl, lm);
        };
        for (uint32_t t = 0; t < obmt::NT; t++) {
            uint32_t nl[obmt::WPT], sp[obmt::WPT], lm[obmt::WPT];
            load(t, nl, sp, lm);
            uint32_t c0 = obmt::first_events(nl, sp, lm, 0, nullptr), c1 = obmt::first_events(nl, sp, lm, 1, nullptr);
            g[t] = c0 != 0; pr[t] = (c1 != 0 && c0 == 0);
        }
        uint32_t warp_cin = 0, naive = 0;
        for (uint32_t w = 0; w < obmt::NT / 32; w++) {
            uint32_t Gb = 0, Pb = 0;
            for (uint32_t l = 0; l < 32; l++) { Gb |= g[w * 32 + l] << l; Pb |= pr[w * 32 + l] << l; }
            uint32_t w0, w1, cout;
            obmt::carry_lookahead32(Gb, Pb, 0, &w0);
            obmt::carry_lookahead32(Gb, Pb, 1, &w1);
            uint32_t C = obmt::carry_lookahead32(Gb, Pb, warp_cin, &cout);
            for (uint32_t l = 0; l < 32; l++) {
                cin_t[w * 32 + l] = (C >> l) & 1u;
                if (cin_t[w * 32 + l] != naive) { fprintf(stderr, "hostsim: carry look-ahead mismatch at thread %u\n", w * 32 + l); abort(); }
                naive = g[w * 32 + l] | (pr[w * 32 + l] & naive); /* sequential reference */
            }
            uint32_t f = w0 | ((w1 & ~w0 & 1u) << 1);
            warp_cin = (f & 1u) | ((f >> 1) & warp_cin);
            if (warp_cin != cout) { fprintf(stderr, "hostsim: warp carry mismatch\n"); abort(); }
        }
        uint32_t n_owners = 0;
        for (uint32_t t = 0; t < obmt::NT; t++) {
            uint32_t nl[obmt::WPT], sp[obmt::WPT], lm[obmt::WPT];
            load(t, nl, sp, lm);
            obmt::first_events(nl, sp, lm, cin_t[t], &lbs[t]);
            my_nl[t] = my_own[t] = 0;
            for (uint32_t j = 0; j < obmt::WPT; j++) { my_own[t] += (uint32_t)__builtin_popcount(lbs[t].own[j]); my_nl[t] += (uint32_t)__builtin_popcount(nl[j]); }
            n_owners += my_own[t];
        }
        uint32_t nlp = 0, own = 0;
        for (uint32_t t = 0; t < obmt::NT; t++) {
            uint32_t q = nlp;
            for (uint32_t j = 0; j < obmt::WPT; j++) { S.nlpre[t * obmt::WPT + j] = (uint16_t)q; q += (uint32_t)__builtin_popcount(S.nlw[t * obmt::WPT + j]); }
            if (n_owners <= obmt::QMAX) {
                uint32_t o = own;
                for (uint32_t j = 0; j < obmt::WPT; j++) {
                    uint32_t bits = lbs[t].own[j];
                    while (bits) { S.owner[o++] = (t * obmt::WPT + j) * 32 + (uint32_t)__builtin_ctz(bits); bits &= bits - 1; }
                }
            }
            nlp += my_nl[t]; own += my_own[t];
        }
        S.n_owners = n_owners <= obmt::QMAX ? n_owners : 0;
        S.n_markers_q = 0;
        if (n_owners > obmt::QMAX) for (uint32_t t = 0; t < nd; t++) S.dflag[t] |= obmt::DF_QOVERFLOW;
        n_owners = S.n_owners;
        return n_owners;
    }
    uint32_t count(const uint8_t *bytes, const uint64_t *doc_off, uint32_t da, uint32_t db, uint32_t fake_skew) {
        const uint32_t nd = db - da;
        uint32_t n_owners = scan(bytes, doc_off, da, db, fake_skew);
        /* the device fills mlist in a nondeterministic order: emulate an adversarial one (reverse) */
        for (uint32_t o = n_owners; o-- > 0;) obmt::owner_prepare(S, o);
        for (uint32_t m = 0; m < S.n_markers_q; m++) obmt::marker_stage(S, TBL, m);
        uint32_t e = 0;
        for (uint32_t o = 0; o < obmt::QMAX; o++) {
            uint32_t v = (o < n_owners && !S.dflag[S.odoc[o] & 0x7Fu]) ? S.ocnt[o] : 0;
            S.ocnt[o] = e; e += v;
        }
        S.ocnt[obmt::QMAX] = e;
        if (n_owners < obmt::QMAX) S.ocnt[n_owners] = e;
        for (uint32_t t = 0; t <= nd; t++) S.dfirst[t] = t == nd ? n_owners : obmt::first_owner_at(S, S.dstart[t]);
        for (uint32_t t = 0; t < nd; t++) obmt::doc_count(S, TBL, t);
        uint32_t acc = 0;
        for (uint32_t t = 0; t < nd; t++) { uint32_t v = S.dcnt[t]; S.dcnt[t] = acc; acc += v; }
        S.dcnt[nd] = acc; sub_total = acc;
        return acc;
    }
    void fill(uint32_t da, uint32_t db, uint64_t base, obm_tuple *out, uint64_t cap, uint64_t *tuple_off, obmt::FillStats &fs) {
        for (uint32_t o = 0; o < S.n_owners; o++) obmt::owner_fill_thread(S, TBL, o, S.ocnt[o + 1] - S.ocnt[o], out, cap, base, fs);
        uint32_t nm = S.n_markers_q < obmt::NSTAGE ? S.n_markers_q : obmt::NSTAGE;
        for (uint32_t m = 0; m < nm; m++) for (uint32_t lane = 0; lane < 32; lane++) obmt::owner_fill_staged(S, m, lane, 32, out, cap, base, fs);
        for (uint32_t t = 0; t < db - da; t++) { tuple_off[da + t] = base + S.dcnt[t]; obmt::doc_fill(S, TBL, t, out, cap, base, fs); }
    }
};
} // namespace

extern "C" uint64_t hs_tile_batch(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, obm_tuple *out, uint64_t cap,
                                  uint64_t *tuple_off, uint32_t fake_skew, uint64_t *stats /* markers, lexemes, exact, fatal */) {
    static Emu emu;
    const uint64_t total = doc_off[ndocs];
    emu.total_bytes = total;
    const uint64_t ntiles = total / obmt::TILE + 1;
    uint64_t base = 0;
    obmt::FillStats fs = {0, 0, 0, 0};
    uint32_t d = 0;
    for (uint64_t t = 0; t < ntiles; t++) {
        uint32_t d_first = d;
        while (d < ndocs && doc_off[d] < (t + 1) * (uint64_t)obmt::TILE) d++;
        uint32_t d_last = d, d_small_end = d_last;
        bool large = d_last > d_first && doc_off[d_last] - doc_off[d_last - 1] > obmt::MAXDOC;
        if (large) d_small_end = d_last - 1;
        for (uint32_t da = d_first; da < d_small_end; da += obmt::DMAX) {
            uint32_t db = da + obmt::DMAX < d_small_end ? da + obmt::DMAX : d_small_end;
            uint32_t sub = emu.count(bytes, doc_off, da, db, fake_skew);
            emu.fill(da, db, base, out, cap, tuple_off, fs);
            base += sub;
        }
        if (large) {
            uint32_t dl = d_last - 1;
            tuple_off[dl] = base;
            obm::WriteSink sink(out + base, base < cap ? cap - base : 0);
            obm::Lexer<obm::WriteSink> lx(TBL, bytes + doc_off[dl], (uint32_t)(doc_off[dl + 1] - doc_off[dl]), sink);
            int st = lx.run<false>();
            fs.markers += sink.n_markers; fs.lexemes += sink.n_lexemes; fs.exact_docs++; fs.fatal_docs += st == obm::RUN_FATAL;
            base += sink.n_tuples;
        }
    }
    tuple_off[ndocs] = base;
    if (stats) { stats[0] = fs.markers; stats[1] = fs.lexemes; stats[2] = fs.exact_docs; stats[3] = fs.fatal_docs; }
    return base;
}


/* ---------------------------------------------------------------------------------------------
 * Emulation of the two-stage pipeline (obm_pipe.cuh): k1_scan builds per-unit item runs with EOF
 * items and unit records; k2_units is replayed unit by unit (one warp each on the device) with the
 * same block structure, staging capacity, look-up sentinel and flag handling as the kernel.
 * ------------------------------------------------------------------------------------------- */
namespace {
struct PipeEmu {
    const uint8_t *bytes; const uint64_t *doc_off; obm_tuple *out; uint64_t cap; uint64_t *tuple_off;
    std::vector<obmp::item_t> items; std::vector<obmp::Unit> units; std::vector<uint32_t> doc_flag, counts;
    uint64_t st_m = 0, st_l = 0, st_e = 0, st_f = 0;
    /* per-warp shared memory */
    obm_tuple stage[obmp::W_MLCAP * obmp::W_LTS]; uint64_t moff[obmp::W_MLCAP]; uint16_t icnt[obmp::W_ICAP]; uint8_t mlist[obmp::W_ICAP];
    uint64_t i0; uint32_t d0, nd; uint64_t total_bytes = 0; uint64_t views = 0, unsafe_views = 0;
    uint32_t doc_of(obmp::item_t it) const { return obmp::it_large(it) ? d0 + nd : d0 + obmp::it_doc(it); }
    uint32_t dlen(uint32_t d) const { return (uint32_t)(doc_off[d + 1] - doc_off[d]); }
    /* k2_lex_lines: up to 32 lines (one per lane) with their text packed into the pool; everything outside the copied
     * chunks is poison, so any dependence on bytes past a view shows up */
    void lex_lines(uint32_t kn, const obmp::item_t *its, const uint32_t *ds, obm_tuple *const *outs, const uint32_t *caps, uint32_t *rs,
                   uint32_t *mk, uint32_t *lx) {
        using namespace obmp;
        alignas(16) static uint8_t pool[W_POOL * 16];
        memset(pool, 0x2B, sizeof pool);
        uint32_t pool_used = 0;
        for (uint32_t q = 0; q < kn; q++) {
            const uint32_t d = ds[q]; item_t it = its[q];
            const uint8_t *doc = bytes + doc_off[d]; uint32_t n_view = dlen(d);
            if (it_unicode(it)) { rs[q] = k2_unicode_item(TBL, doc, n_view, it, outs[q], caps[q], mk, lx); continue; }
            LineView v = line_view(bytes + doc_off[d], dlen(d), it, bytes, total_bytes);
            const uint32_t want = v.nch <= 32u ? v.nch : 0u;
            pool_used += want; /* the scan is over all lines, fitting or not, exactly like the warp scan */
            if (want && pool_used <= W_POOL) {
                uint8_t *sm = pool + (size_t)(pool_used - want) * 16u;
                memcpy(sm, (const void *)v.g0, (size_t)want * 16u);
                const uint32_t nv = line_view_safe(sm, v, bytes + doc_off[d], dlen(d), it);
                if (nv) { doc = sm + (intptr_t)((uintptr_t)(bytes + doc_off[d]) - v.g0); n_view = nv; views++; } else unsafe_views++;
            }
            rs[q] = k2_marker_item(TBL, doc, n_view, it, outs[q], caps[q], mk, lx);
        }
    }
    bool lex_block(uint32_t b0, uint32_t b1, bool stable, uint32_t &n_ml_out) {
        using namespace obmp;
        uint32_t n_ml = 0; bool any = false;
        for (uint32_t k = 0; k < W_MLCAP; k++) moff[k] = ~0ull;
        for (uint32_t i = b0; i < b1; i++) {
            item_t it = items[i0 + i];
            bool m = it_marker(it);
            if (stable && doc_flag[doc_of(it)]) { m = false; icnt[i - b0] = it_eof(it) ? G_CNT_LOOKUP : (uint16_t)0; }
            else if (!m) {
                if (it_exact(it) || it_large(it)) { icnt[i - b0] = G_CNT_LOOKUP; any = true; }
                else icnt[i - b0] = (uint16_t)simple_count(it);
            }
            if (m) mlist[n_ml++] = (uint8_t)(i - b0);
        }
        /* lines are lexed in rounds of 32 (one per lane); every round packs its text into the pool */
        for (uint32_t k0 = 0; k0 < n_ml; k0 += 32) {
            const uint32_t kn = n_ml - k0 < 32 ? n_ml - k0 : 32;
            item_t its[32]; uint32_t ds[32], rs[32]; obm_tuple *outs[32]; uint32_t caps[32];
            for (uint32_t q = 0; q < kn; q++) {
                its[q] = items[i0 + b0 + mlist[k0 + q]]; ds[q] = doc_of(its[q]);
                outs[q] = k0 == 0 ? stage + q * W_LTS : nullptr; caps[q] = k0 == 0 ? W_LTS : 0u;
            }
            lex_lines(kn, its, ds, outs, caps, rs, nullptr, nullptr);
            for (uint32_t q = 0; q < kn; q++) {
                const uint32_t ib = mlist[k0 + q], d = ds[q], r = rs[q];
                icnt[ib] = (uint16_t)mres_tuples(r);
                if (mres_irregular(r)) { doc_flag[d] |= GF_INTERACT; any = true; }
            }
        }
        n_ml_out = n_ml;
        return any;
    }
    void count_flagged_docs() {
        for (uint32_t q = 0; q < nd; q++) {
            const uint32_t d = d0 + q, f = doc_flag[d];
            if (f && !(f & obmp::GF_LARGE)) { obm::SmallSink s(nullptr, 0); obmp::doc_exact(TBL, bytes + doc_off[d], dlen(d), s); counts[d] = s.n_tuples; }
        }
    }
    void apply_flags(uint32_t b0, uint32_t b1) {
        for (uint32_t i = b0; i < b1; i++) { obmp::item_t it = items[i0 + i]; if (doc_flag[doc_of(it)]) icnt[i - b0] = obmp::it_eof(it) ? obmp::G_CNT_LOOKUP : (uint16_t)0; }
    }
    uint64_t block_total(uint32_t b0, uint32_t b1) {
        uint64_t sum = 0;
        for (uint32_t i = b0; i < b1; i++) { uint32_t c = icnt[i - b0]; if (c == obmp::G_CNT_LOOKUP) c = counts[doc_of(items[i0 + i])]; sum += c; }
        return sum;
    }
    void flush_relex(std::vector<obmp::item_t> &its, std::vector<uint32_t> &ds, std::vector<uint64_t> &ats) {
        if (its.empty()) return;
        obm_tuple *outs[32]; uint32_t caps[32], rs[32], mk = 0, lx = 0;
        for (size_t q = 0; q < its.size(); q++) { outs[q] = out + ats[q]; caps[q] = ats[q] < cap ? (uint32_t)(cap - ats[q]) : 0u; }
        lex_lines((uint32_t)its.size(), its.data(), ds.data(), outs, caps, rs, &mk, &lx);
        st_m += mk; st_l += lx;
        its.clear(); ds.clear(); ats.clear();
    }
    uint64_t write_block(uint32_t b0, uint32_t b1, uint32_t n_ml, uint64_t at0, bool stable) {
        using namespace obmp;
        uint64_t at = at0; uint32_t k = 0;
        std::vector<item_t> relex_it; std::vector<uint32_t> relex_d; std::vector<uint64_t> relex_at;
        for (uint32_t i = b0; i < b1; i++) {
            if (((i - b0) & 31u) == 0) flush_relex(relex_it, relex_d, relex_at); /* the kernel re-lexes per 32-item chunk */
            item_t it = items[i0 + i];
            uint32_t c = icnt[i - b0]; const bool lookup = c == G_CNT_LOOKUP;
            const uint32_t d = doc_of(it);
            if (lookup) c = counts[d];
            if (it_marker(it) && !(stable && doc_flag[d])) { /* same membership rule as lex_block's mlist */
                if (c) {
                    if (k < W_MLCAP && c <= W_LTS) moff[k] = at;
                    else { relex_it.push_back(it); relex_d.push_back(d); relex_at.push_back(at); }
                }
                k++;
            } else if (it_marker(it)) {
                /* line of a flagged document: nothing to write */
            } else if (it_eof(it)) {
                tuple_off[d + 1] = at + c;
                if (!lookup) { if (at < cap) out[at] = OBM_TUPLE(OBM_K_EOF, it_ls(it), 0); st_l++; }
                else if (it_large(it)) { /* k_exact_fill on the device */
                    obm::WriteSink sink(out + at, at < cap ? cap - at : 0);
                    obm::Lexer<obm::WriteSink> lx(TBL, bytes + doc_off[d], dlen(d), sink);
                    lx.run<false>();
                } else {
                    obm::SmallSink s(out + at, at < cap ? (uint32_t)(cap - at) : 0u);
                    int st = doc_exact(TBL, bytes + doc_off[d], dlen(d), s);
                    st_m += s.n_markers; st_l += s.n_lexemes; st_e++; st_f += st == obm::RUN_FATAL;
                }
            } else if (c) { plain_write(it, out, at, cap); st_l++; }
            at += c;
        }
        flush_relex(relex_it, relex_d, relex_at);
        for (uint32_t q = 0; q < (n_ml < W_MLCAP ? n_ml : W_MLCAP); q++) {
            if (moff[q] == ~0ull) continue;
            const uint32_t c = icnt[mlist[q]];
            for (uint32_t l = 0; l < c; l++) {
                obm_tuple tup = stage[q * W_LTS + l];
                if (moff[q] + l < cap) out[moff[q] + l] = tup;
                uint32_t kind = OBM_TUPLE_KIND(tup);
                st_m += kind == OBM_K_MARKER_START; st_l += (kind - (uint32_t)OBM_K_PART) > 4u;
            }
        }
        return at - at0;
    }
};
} // namespace

extern "C" uint64_t hs_pipe_batch(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, obm_tuple *out, uint64_t cap,
                                   uint64_t *tuple_off, uint32_t fake_skew, uint64_t *stats) {
    static Emu emu; emu.uni_lines = true; emu.total_bytes = doc_off[ndocs];
    using namespace obmp;
    PipeEmu G; G.bytes = bytes; G.doc_off = doc_off; G.out = out; G.cap = cap; G.tuple_off = tuple_off;
    G.doc_flag.assign(ndocs, 0); G.counts.assign(ndocs, 0);
    const uint64_t total = doc_off[ndocs];
    G.total_bytes = total;
    const uint64_t ntiles = total / obmt::TILE + 1;
    /* K1 */
    uint32_t d = 0;
    for (uint64_t t = 0; t < ntiles; t++) {
        uint32_t d_first = d;
        while (d < ndocs && doc_off[d] < (t + 1) * (uint64_t)obmt::TILE) d++;
        uint32_t d_last = d;
        if (d_last == d_first) continue;
        const bool has_large = doc_off[d_last] - doc_off[d_last - 1] > obmt::MAXDOC;
        const uint32_t d_small_end = d_last - (has_large ? 1u : 0u);
        uint32_t nsub = (d_small_end - d_first + obmt::DMAX - 1) / obmt::DMAX; if (nsub == 0) nsub = 1;
        if (has_large) {
            const uint32_t dl = d_last - 1; G.doc_flag[dl] = GF_LARGE;
            obm::SmallSink s(nullptr, 0); obm::Lexer<obm::SmallSink> lx(TBL, bytes + doc_off[dl], (uint32_t)(doc_off[dl + 1] - doc_off[dl]), s);
            int st = lx.run<false>(); G.counts[dl] = s.n_tuples; G.st_m += s.n_markers; G.st_l += s.n_lexemes; G.st_e++; G.st_f += st == obm::RUN_FATAL;
        }
        for (uint32_t k = 0; k < nsub; k++) {
            const uint32_t da = d_first + k * obmt::DMAX, db = da + obmt::DMAX < d_small_end ? da + obmt::DMAX : d_small_end, nd = db - da;
            const uint32_t extra = (k == nsub - 1 && has_large) ? 1u : 0u;
            uint32_t n_owners = 0;
            std::vector<item_t> sit;
            if (nd) {
                emu.scan(bytes, doc_off, da, db, fake_skew);
                n_owners = emu.S.n_owners;
                sit.resize(n_owners);
                for (uint32_t o = 0; o < n_owners; o++) sit[o] = k1_owner_item(emu.S, o);
            }
            std::vector<uint32_t> lp(n_owners + 1, 0); /* live owners before o (dead lines own no tuple and are dropped) */
            for (uint32_t o = 0; o < n_owners; o++) lp[o + 1] = lp[o] + (it_dead(sit[o]) ? 0u : 1u);
            const uint32_t n_items = lp[n_owners] + nd + extra;
            const uint64_t ibase = G.items.size();
            G.items.resize(ibase + n_items, ~0ull);
            for (uint32_t o = 0; o < n_owners; o++) if (!it_dead(sit[o])) G.items[ibase + lp[o] + it_doc(sit[o])] = sit[o];
            for (uint32_t q = 0; q < nd; q++) {
                uint32_t lo = 0; while (lo < n_owners && it_doc(sit[lo]) <= q) lo++;
                lo = lp[lo];
                const uint32_t f = emu.S.dflag[q];
                G.doc_flag[da + q] = ((f & obmt::DF_NONASCII) ? GF_NONASCII : 0u) | ((f & obmt::DF_QOVERFLOW) ? GF_QOVERFLOW : 0u);
                G.items[ibase + lo + q] = make_eof_item(emu.S.dstart[q + 1] - emu.S.dstart[q], q, (f & obmt::DF_EXACT_MASK) != 0);
            }
            if (extra) G.items[ibase + n_items - 1] = make_large_item();
            for (uint64_t i = ibase; i < ibase + n_items; i++) if (G.items[i] == ~0ull) { fprintf(stderr, "hostsim: item hole\n"); abort(); }
            if (getenv("HS_DUMP_ITEMS")) for (uint64_t i = ibase; i < ibase + n_items; i++) fprintf(stderr, "item %llu: marker=%d uni=%d eof=%d dead=%d doc=%u ls=%u pos=%u line=%u le=%u dflag=%u\n", (unsigned long long)i, (int)it_marker(G.items[i]), (int)it_unicode(G.items[i]), (int)it_eof(G.items[i]), (int)it_dead(G.items[i]), it_doc(G.items[i]), it_ls(G.items[i]), it_pos(G.items[i]), it_line(G.items[i]), it_marker(G.items[i]) ? it_line_end(G.items[i]) : 0u, emu.S.dflag[it_doc(G.items[i]) < nd ? it_doc(G.items[i]) : 0]);
            G.units.push_back(Unit{ibase, da, n_items | (nd << 16)});
        }
    }
    /* K2: units in id order (the look-back chain) */
    uint64_t base = 0;
    tuple_off[0] = 0;
    for (const Unit &U : G.units) {
        const uint32_t n_items = unit_items(U);
        G.i0 = U.item_base; G.d0 = U.doc_base; G.nd = unit_nd(U);
        uint32_t n_ml = 0;
        if (n_items <= W_ICAP) {
            if (G.lex_block(0, n_items, false, n_ml)) { G.count_flagged_docs(); G.apply_flags(0, n_items); }
            base += G.write_block(0, n_items, n_ml, base, false);
        } else {
            uint64_t total_u = 0; bool any = false;
            for (uint32_t b0 = 0; b0 < n_items; b0 += 32) { uint32_t nm, b1 = b0 + 32 < n_items ? b0 + 32 : n_items; any |= G.lex_block(b0, b1, false, nm); total_u += G.block_total(b0, b1); }
            if (any) {
                G.count_flagged_docs();
                total_u = 0;
                for (uint32_t b0 = 0; b0 < n_items; b0 += 32) { uint32_t nm, b1 = b0 + 32 < n_items ? b0 + 32 : n_items; G.lex_block(b0, b1, true, nm); total_u += G.block_total(b0, b1); }
            }
            uint64_t at = base;
            for (uint32_t b0 = 0; b0 < n_items; b0 += 32) { uint32_t nm, b1 = b0 + 32 < n_items ? b0 + 32 : n_items; G.lex_block(b0, b1, true, nm); at += G.write_block(b0, b1, nm, at, true); }
            if (at - base != total_u) { fprintf(stderr, "hostsim: large-unit sweeps disagree (%llu vs %llu)\n", (unsigned long long)(at - base), (unsigned long long)total_u); abort(); }
            base = at;
        }
    }
    tuple_off[ndocs] = base;
    if (stats) { stats[0] = G.st_m; stats[1] = G.st_l; stats[2] = G.st_e; stats[3] = G.st_f; }
    if (getenv("HS_VIEW_STATS")) fprintf(stderr, "hostsim: %llu staged line views, %llu rejected\n", (unsigned long long)G.views, (unsigned long long)G.unsafe_views);
    return base;
}

/* ---------------------------------------------------------------------------------------------
 * Large documents: the chunk-parallel exact path (obm_large.h), replayed sequentially with the same
 * chain check and the same fallback as k_large_count / k_large_resolve / k_large_fill.
 * returns the tuple count; *used_chunks = 1 when the chain validated (no sequential fallback)
 * ------------------------------------------------------------------------------------------- */
#include "../../operator-builder_b200/csrc/obm_large.h"
/* k_large_prep + k_large_lines: the resolved start and line of every chunk (cs and line hold n_chunks(n) entries) */
extern "C" uint32_t hs_large_chunk_starts(const uint8_t *doc, uint32_t n, uint32_t *cs, uint32_t *line) {
    using namespace obml;
    const uint32_t nc = n_chunks(n);
    uint32_t acc = 0;
    for (uint32_t c = 0; c < nc; c++) { uint32_t sk; cs[c] = chunk_start(doc, n, c, &sk); line[c] = 1 + acc + sk; acc += chunk_newlines(doc, n, c); }
    resolve_chunk_starts(cs, line, nc);
    return nc;
}
extern "C" uint64_t hs_large_doc(const uint8_t *doc, uint32_t n, obm_tuple *out, uint64_t cap, uint32_t *used_chunks) {
    using namespace obml;
    const uint32_t nc = n_chunks(n);
    std::vector<uint32_t> cs(nc + 1), line(nc), cnt(nc), cend(nc), flag(nc);
    hs_large_chunk_starts(doc, n, cs.data(), line.data());
    cs[nc] = n;
    bool valid = true, ascii = true;
    for (uint32_t c = 0; c < nc; c++) ascii = ascii && !chunk_non_ascii(doc, n, c);
    for (uint32_t c = 0; c < nc; c++) {
        obm::SmallSink s(nullptr, 0);
        flag[c] = ascii ? lex_chunk<obm::SmallSink, true>(TBL, doc, n, cs[c], line[c], cs[c + 1], s, &cend[c])
                        : lex_chunk<obm::SmallSink, false>(TBL, doc, n, cs[c], line[c], cs[c + 1], s, &cend[c]);
        cnt[c] = s.n_tuples;
        if (flag[c] || cend[c] != cs[c + 1]) valid = false;
    }
    if (used_chunks) *used_chunks = valid;
    if (!valid) return hs_lex_doc(doc, n, out, cap, nullptr, nullptr);
    uint64_t at = 0;
    for (uint32_t c = 0; c < nc; c++) {
        obm::WriteSink s(out + at, at < cap ? cap - at : 0);
        uint32_t e;
        if (ascii) lex_chunk<obm::WriteSink, true>(TBL, doc, n, cs[c], line[c], cs[c + 1], s, &e);
        else lex_chunk<obm::WriteSink, false>(TBL, doc, n, cs[c], line[c], cs[c + 1], s, &e);
        if (s.n_tuples != cnt[c]) { fprintf(stderr, "hostsim: chunk count changed between passes\n"); abort(); }
        at += cnt[c];
    }
    if (at < cap) out[at] = OBM_TUPLE(OBM_K_EOF, n, 0);
    return at + 1;
}

/* utf8_plain (obm_tile.h) on one document staged the way k1_scan stages it: 1 = valid UTF-8 without Unicode white space */
extern "C" int hs_utf8_plain(const uint8_t *doc, uint32_t n, uint32_t fake_skew) {
    static Emu emu;
    if (n > obmt::MAXDOC) return -1;
    const uint64_t off[2] = {0, n};
    emu.uni_lines = true; emu.total_bytes = n;
    emu.scan(doc, off, 0, 1, fake_skew);
    return (emu.S.dflag[0] & obmt::DF_NONASCII) ? 0 : 1; /* ASCII documents are trivially plain */
}

/* ---------------------------------------------------------------------------------------------
 * The fused warp kernel (csrc/obm_warp_core.h, mode 0): the device source itself, compiled for the host and run by
 * 32 fibers per warp (warp_emu.h).  Units are processed in id order, which is what the look-back chain enforces.
 * ------------------------------------------------------------------------------------------- */
#include "warp_emu.h"
struct uint4 { uint32_t x, y, z, w; };
#define WLANE() wemu::lane()
#define WBALLOT(p) wemu::ballot((p))
#define WSHFL(v, s) wemu::shfl((uint32_t)(v), (uint32_t)(s))
#define WSHFL_UP(v, d) wemu::shfl_up((uint32_t)(v), (uint32_t)(d))
#define WSYNC() wemu::sync()
#define WTEXT(S) ((const uint8_t *)(S).text)
#define WATOMIC_OR(p, v) (*(p) |= (v))
static uint64_t g_wstat_fast = 0, g_wstat_generic = 0;
#define OBMW_STAT(name) (g_wstat_##name++)
#include "../../operator-builder_b200/csrc/obm_warp_core.h"
extern "C" void hs_warp_line_stats(uint64_t *fast, uint64_t *generic) { *fast = g_wstat_fast; *generic = g_wstat_generic; }


namespace {
/* bytes that a read of dead text would turn into tuples: line starts, markers, comments, scopes, values, an unterminated
 * back-tick string, and bytes >= 0x80 (the exact lexer) -- in a phase that shifts from one staging to the next */
const uint8_t POISON[] = {'\n', '+', '#', '/', ':', '=', '`', 0x80, 0xff};
struct HostHooks {
    const uint64_t *doc_off = nullptr;
    uint32_t da = 0, nd = 0, skew = 0; /* the unit being scanned: what compute_unit must have put in W.dstart */
    uint32_t shift = 0;
    uint64_t bad_starts = 0;
    void poison(obmw::WarpSmem &S) {
        for (size_t i = 0; i < sizeof S.text; i++) S.text[i] = POISON[(i + shift) % sizeof POISON];
        shift++;
    }
    /* the device's bulk copy, landed at once over text that is dead by the pipeline's rules */
    void stage(obmw::WarpSmem &S, const void *gsrc, uint32_t nbytes) {
        if (wemu::lane() == 0) { poison(S); memcpy(S.text, gsrc, nbytes); }
    }
    /* compute_unit has written the document starts (from D.doff when prestaged): check them against doc_off, and put the
     * right ones in place so that a wrong start is reported instead of sending the scan outside the buffer */
    void stage_wait(obmw::WarpSmem &S, uint32_t) {
        const uint32_t l = wemu::lane();
        if (l > nd) return;
        const uint32_t want = (uint32_t)(doc_off[da + l] - doc_off[da]) + skew;
        if (S.dstart[l] != want) {
            if (bad_starts++ < 4) fprintf(stderr, "hostsim: documents [%u, %u]: dstart[%u] = %u, doc_off gives %u\n", da, da + nd, l, S.dstart[l], want);
            S.dstart[l] = want;
        }
    }
};
}

/* one row of hs_warp_batch_report per unit, in unit order */
enum { WREP_U, WREP_DA, WREP_ND, WREP_EXTRA, WREP_NEEDS_TEXT, WREP_PAGED, WREP_DEFERRED, WREP_OVER_FIN, WREP_LONG_LINE, WREP_PRESTAGED, WREP_N };

/* The software pipeline of k_warp_scan, in its order, by one warp that takes every unit in id order (which is what the
 * look-back chain enforces): scan unit i, publish its count, take unit i + 1's descriptor and -- where prestage_next allows
 * it -- stage its text at once over unit i's and load its document offsets lane by lane, then write unit i - 1 from
 * W.fin, then assemble unit i into W.fin or write it directly.  Large documents are counted before the loop (the side
 * stream) and filled after it.  Returns the tuple count, or ~0 when a unit's document starts were wrong. */
extern "C" uint64_t hs_warp_batch_report(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, obm_tuple *out, uint64_t cap,
                                         uint64_t *tuple_off, uint64_t *stats, uint32_t *report, uint64_t report_cap, uint64_t *n_units) {
    using namespace obmw;
    static WarpSmem S; static wemu::Warp W; static bool poisoned = false;
    if (!poisoned) { memset(&S, 0x2B, sizeof S); poisoned = true; }
    const uint64_t total = doc_off[ndocs];
    const uint64_t ntiles = total / TILE + 1;
    std::vector<uint32_t> counts(ndocs + 1, 0);
    uint32_t status[4] = {0, 0, 0, 0}; unsigned long long totals[2] = {0, 0};
    WArgs A; memset(&A, 0, sizeof A);
    A.bytes = bytes; A.doc_off = doc_off; A.ndocs = ndocs; A.total_bytes = total; A.ntiles = (uint32_t)ntiles;
    A.counts = counts.data(); A.out = out; A.out_cap = cap; A.tuple_off = tuple_off; A.status = status; A.totals = totals;
    /* k_wtile_index, k_wunits, the scan, k_wunit_descs */
    std::vector<WRec> recs(ntiles); std::vector<uint64_t> ubase(ntiles + 1, 0);
    uint32_t d = 0;
    for (uint64_t t = 0; t < ntiles; t++) {
        const uint32_t d0 = d;
        while (d < ndocs && doc_off[d] < (t + 1) * (uint64_t)TILE) d++;
        recs[t] = make_wrec(doc_off, d0, d);
        ubase[t + 1] = ubase[t] + recs[t].n_units;
    }
    const uint32_t nunits = (uint32_t)ubase[ntiles];
    std::vector<WUnit> units(nunits);
    for (uint64_t t = 0; t < ntiles; t++)
        for (uint32_t k = 0; k < recs[t].n_units; k++) units[ubase[t] + k] = make_wunit(doc_off, recs[t], k);
    A.ubase = ubase.data(); A.units = units.data();
    if (n_units) *n_units = nunits;
    uint64_t st_m = 0, st_l = 0, st_e = 0, st_f = 0, chain = 0;
    /* k_large_count: every large document before the scan */
    std::vector<uint32_t> large_docs;
    for (const WUnit &w : units) {
        if (!wu_extra(w)) continue;
        const uint32_t dl = w.da + wu_nd(w);
        obm::SmallSink s(nullptr, 0); obm::Lexer<obm::SmallSink> lx(TBL, bytes + doc_off[dl], (uint32_t)(doc_off[dl + 1] - doc_off[dl]), s);
        const int st = lx.run<false>(); counts[dl] = s.n_tuples; st_m += s.n_markers; st_l += s.n_lexemes; st_e++; st_f += st == obm::RUN_FATAL;
        large_docs.push_back(dl);
    }
    HostHooks H; H.doc_off = doc_off;
    auto add_acc = [&](WAcc *a) { for (int l = 0; l < 32; l++) { st_m += a[l].markers; st_l += a[l].lexemes; st_e += a[l].exact; st_f += a[l].fatal; } };
    /* the descriptor of unit u as every lane holds it (doff: not loaded) */
    auto unit_desc = [&](uint32_t u, UnitDesc *D) {
        for (int l = 0; l < 32; l++) {
            if (u < nunits) D[l] = make_desc(A, u, units[u]);
            else { D[l] = UnitDesc{0, 0, 0, 0, 0, 0, 0, false, 0}; }
        }
    };
    UnitRegs pend[32]; bool have_pend = false;
    uint64_t pend_base = 0;
    UnitDesc cur[32], nxt[32];
    unit_desc(0, cur);
    bool prestaged = false;
    while (cur[0].valid) {
        UnitRegs R[32];
        H.da = cur[0].da; H.nd = cur[0].db - cur[0].da; H.skew = cur[0].skew;
        wemu::run(W, [&]() { compute_unit(S, S.set, A, TBL, H, cur[wemu::lane()], prestaged, R[wemu::lane()]); });
        const uint64_t my_base = chain; chain += R[0].total; /* publish */
        unit_desc(cur[0].u + 1, nxt);
        const bool pre = prestage_next(R[0], nxt[0]);
        if (pre) { /* the next unit's bulk copy, as if it landed at once, and its document offsets, a lane each */
            H.poison(S);
            memcpy(S.text, (const void *)(uintptr_t)nxt[0].base_abs, desc_load(nxt[0]));
            for (uint32_t l = 0; l <= nxt[0].db - nxt[0].da; l++) nxt[l].doff = doc_off[nxt[0].da + l];
        }
        if (have_pend) { wemu::run(W, [&]() { write_fin(S, A, pend[wemu::lane()], nunits, pend_base); }); have_pend = false; }
        WAcc a[32]; memset(a, 0, sizeof a);
        bool deferred[32]; memset(deferred, 0, sizeof deferred);
        if (!R[0].needs_text) wemu::run(W, [&]() { deferred[wemu::lane()] = assemble_fin(S, S.set, R[wemu::lane()], a[wemu::lane()]); });
        if (deferred[0]) { memcpy(pend, R, sizeof R); pend_base = my_base; have_pend = true; }
        else wemu::run(W, [&]() { write_unit(S, S.set, A, TBL, R[wemu::lane()], nunits, my_base, a[wemu::lane()]); });
        add_acc(a);
        const uint32_t u = cur[0].u;
        if (report && u < report_cap) {
            uint32_t *r = report + (uint64_t)u * WREP_N;
            r[WREP_U] = u; r[WREP_DA] = cur[0].da; r[WREP_ND] = R[0].nd; r[WREP_EXTRA] = R[0].extra;
            r[WREP_NEEDS_TEXT] = R[0].needs_text; r[WREP_PAGED] = R[0].paged; r[WREP_DEFERRED] = deferred[0];
            r[WREP_OVER_FIN] = R[0].n_small > FIN_CAP; r[WREP_LONG_LINE] = R[0].long_line; r[WREP_PRESTAGED] = prestaged;
        }
        memcpy(cur, nxt, sizeof cur);
        prestaged = pre;
    }
    if (have_pend) wemu::run(W, [&]() { write_fin(S, A, pend[wemu::lane()], nunits, pend_base); });
    for (uint32_t dl : large_docs) { /* k_large_fill */
        const uint64_t at = tuple_off[dl];
        obm::WriteSink sink(out + at, at < cap ? cap - at : 0);
        obm::Lexer<obm::WriteSink> lx(TBL, bytes + doc_off[dl], (uint32_t)(doc_off[dl + 1] - doc_off[dl]), sink);
        lx.run<false>();
    }
    if (ndocs == 0) tuple_off[0] = 0;
    if (stats) { stats[0] = st_m; stats[1] = st_l; stats[2] = st_e; stats[3] = st_f; }
    return H.bad_starts ? ~0ull : chain;
}
extern "C" uint64_t hs_warp_batch(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, obm_tuple *out, uint64_t cap,
                                  uint64_t *tuple_off, uint32_t fake_skew, uint64_t *stats) {
    (void)fake_skew; /* the skew is the batch's address (tests/hostsim/__init__.py) */
    return hs_warp_batch_report(bytes, doc_off, ndocs, out, cap, tuple_off, stats, nullptr, 0, nullptr);
}
/* ---------------------------------------------------------------------------------------------
 * The phase C stepper alone (tests/test_marker_lines.py): obmw::fast_line on every marker line of each document, from a
 * 16-byte aligned buffer that holds the document at its skew with the staged text's 16 bytes of slack behind it (BUFB -
 * MAXDOC), poisoned around.  The owning lines, their first special ('#', "//" or '+') and first '+' are found as phase B
 * finds them, by a plain byte loop instead of the bitmaps; a '+' PD_GENERIC or more bytes after the first special is the
 * generic lexer's, as in the kernel.  Every marker line runs once into a DirectSink and once into a PackSink(cap = LTS).
 * Per document, out of info[6 * d ...]:
 *   [0] FLR_OK: every marker line on the stepper; FLR_FALLBACK: at least one handed over; FLR_NONE: no marker line
 *   [1] marker lines, [2] of them on the stepper, [3] some stepper line overflowed its PackSink (ovf)
 *   [4] most tuples of one stepper line, [5] largest len of a stepper line's DirectSink tuples
 * direct[toff[d] .. toff[d+1]): the document's tuples (stepper lines from the DirectSink, plain comment lines as phase D
 * writes them) and EOF -- empty when a line was handed over.  staged[soff[d] .. soff[d+1]): the same with the stepper
 * lines' PackSink tuples unpacked -- empty when a line was handed over or overflowed.  Returns 0, or -1 when a document
 * is longer than MAXDOC or an output is too small.
 * ------------------------------------------------------------------------------------------- */
enum { FLR_OK = 0, FLR_FALLBACK = 1, FLR_NONE = 2 };
extern "C" int hs_fast_lines(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, const uint8_t *skews, obm_tuple *direct,
                             uint64_t dcap, uint64_t *toff, obm_tuple *staged, uint64_t scap, uint64_t *soff, uint32_t *info) {
    using namespace obmw;
    alignas(16) static uint8_t buf[BUFB + 64];
    uint32_t pk[LTS];
    uint64_t at = 0, sat = 0;
    toff[0] = 0; soff[0] = 0;
    for (uint32_t d = 0; d < ndocs; d++) {
        const uint32_t n = (uint32_t)(doc_off[d + 1] - doc_off[d]);
        const uint32_t skew = skews[d] & 15u;
        if (n > MAXDOC) return -1;
        for (size_t i = 0; i < sizeof buf; i++) buf[i] = POISON[(i + d) % sizeof POISON];
        memcpy(buf + skew, bytes + doc_off[d], n);
        const uint8_t *t = buf;
        const uint32_t dpos = skew, dend = skew + n;
        uint32_t *inf = info + 6ull * d;
        memset(inf, 0, 6 * sizeof(uint32_t));
        bool fell = false, ovf = false;
        const uint64_t at0 = at, sat0 = sat;
        auto put2 = [&](uint32_t kind, uint32_t off, uint32_t len) {
            if (at < dcap) direct[at] = OBM_TUPLE(kind, off, len);
            if (sat < scap) staged[sat] = OBM_TUPLE(kind, off, len);
            at++; sat++;
        };
        for (uint32_t ls = dpos, line = 1; ls < dend; line++) {
            uint32_t le = ls;
            while (le < dend && t[le] != '\n') le++;
            uint32_t first = ls;
            while (first < le && !(t[first] == '#' || t[first] == '+' || (t[first] == '/' && first + 1 < dend && t[first + 1] == '/'))) first++;
            if (first < le) {
                uint32_t plus = first;
                while (plus < le && t[plus] != '+') plus++;
                if (plus < le) { /* a marker line */
                    inf[1]++;
                    uint32_t res = FL_FALLBACK;
                    if (plus - first < PD_GENERIC) {
                        const uint64_t room = at < dcap ? dcap - at : 0;
                        DirectSink ds(direct + at, room < 0xFFFFFFFFull ? (uint32_t)room : 0xFFFFFFFFu);
                        res = fast_line(t, first, plus, ls, line, dpos, dend, ds);
                        PackSink ps(pk, LTS);
                        const uint32_t res2 = fast_line(t, first, plus, ls, line, dpos, dend, ps);
                        if (res2 != res || ps.n != ds.n || ps.mk != ds.mk || ps.lx != ds.lx) return -2; /* the sinks are passive */
                        if (res == FL_OK) {
                            inf[2]++;
                            if (ds.n > inf[4]) inf[4] = ds.n;
                            for (uint32_t k = 0; k < ds.n && at + k < dcap; k++) {
                                const uint32_t len = (uint32_t)((direct[at + k] >> 32) & 0x7FFFFFFu);
                                if (len > inf[5]) inf[5] = len;
                            }
                            ovf |= ps.ovf;
                            if (!ps.ovf) for (uint32_t k = 0; k < ps.n; k++) { if (sat + k < scap) staged[sat + k] = st_unpack(pk[k]); }
                            at += ds.n; sat += ps.n;
                        }
                    }
                    fell |= res != FL_OK;
                } else { /* a plain comment line */
                    if (line != 1) put2(OBM_K_LINE, ls - dpos, line);
                    put2(OBM_K_COMMENT, first - dpos, t[first] == '/' ? 2 : 1);
                }
            }
            ls = le + 1;
        }
        put2(OBM_K_EOF, n, 0);
        inf[0] = fell ? FLR_FALLBACK : inf[1] ? FLR_OK : FLR_NONE;
        inf[3] = ovf;
        if (fell) at = at0;
        if (fell || ovf) sat = sat0;
        toff[d + 1] = at; soff[d + 1] = sat;
    }
    return at <= dcap && sat <= scap ? 0 : -1;
}

/* units of the batch (k_wunits + the scan): what k_warp_scan's warps share */
extern "C" uint64_t hs_warp_units(const uint64_t *doc_off, uint32_t ndocs) {
    const uint64_t ntiles = doc_off[ndocs] / obmw::TILE + 1;
    uint64_t n = 0;
    uint32_t d = 0;
    for (uint64_t t = 0; t < ntiles; t++) {
        const uint32_t d0 = d;
        while (d < ndocs && doc_off[d] < (t + 1) * (uint64_t)obmw::TILE) d++;
        n += obmw::make_wrec(doc_off, d0, d).n_units;
    }
    return n;
}
