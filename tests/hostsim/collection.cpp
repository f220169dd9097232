/*
 * collection.cpp -- TEST INFRASTRUCTURE.  The collection variant of the fused warp kernel (compute_unit<true> +
 * write_text in csrc/obm_warp_core.h, k_warp_scan<true> on the device), compiled for the host and run by 32 fibers per
 * warp (warp_emu.h), units in id order as the look-back chains enforce.  Beside hostsim.cpp, which replays the plain scan.
 */
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "../../operator-builder_b200/csrc/go_unicode_tables.h"
#include "../../operator-builder_b200/csrc/obm_core.h"

static const char F64[] = GO_F64_OVERFLOW_DIGITS;
static const obm::Tables TBL = { GO_LETTER_RANGES, GO_LETTER_RANGES_N, GO_NUMBER_RANGES, GO_NUMBER_RANGES_N, F64 };

#include "warp_emu.h"
struct uint4 { uint32_t x, y, z, w; };
#define WLANE() wemu::lane()
#define WBALLOT(p) wemu::ballot((p))
#define WSHFL(v, s) wemu::shfl((uint32_t)(v), (uint32_t)(s))
#define WSHFL_UP(v, d) wemu::shfl_up((uint32_t)(v), (uint32_t)(d))
#define WSYNC() wemu::sync()
#define WTEXT(S) ((const uint8_t *)(S).text)
#define WATOMIC_OR(p, v) (*(p) |= (v))
#include "../../operator-builder_b200/csrc/obm_warp_core.h"

namespace {
struct HostHooks {
    void stage(obmw::WarpSmem &S, const void *gsrc, uint32_t nbytes) {
        if (wemu::lane() == 0) memcpy(S.text, gsrc, nbytes); /* whatever the previous unit left behind stays in the buffer, like on the device */
    }
    void stage_wait(obmw::WarpSmem &, uint32_t) {}
    std::vector<uint64_t> *bytes_of_unit = nullptr; /* the byte chain */
    void publish_bytes(uint32_t u, uint64_t n) { if (wemu::lane() == 0) { if (bytes_of_unit->size() <= u) bytes_of_unit->resize(u + 1, ~0ull); (*bytes_of_unit)[u] = n; } }
};
}

/* Manifest.LoadContent's rewrite of one document, as two ReplaceAll passes (the semantics the kernels implement) */
static std::vector<uint8_t> host_rewrite(const uint8_t *p, uint32_t n) {
    auto replace_all = [](const std::vector<uint8_t> &in, const char *pat, const char *rep) {
        const size_t pl = strlen(pat), rl = strlen(rep);
        std::vector<uint8_t> out;
        size_t i = 0;
        while (i < in.size()) {
            if (i + pl <= in.size() && memcmp(in.data() + i, pat, pl) == 0) { out.insert(out.end(), rep, rep + rl); i += pl; }
            else out.push_back(in[i++]);
        }
        return out;
    };
    std::vector<uint8_t> v(p, p + n);
    return replace_all(replace_all(v, "+operator-builder:collection:field", "+operator-builder:field"), "collectionField", "field");
}

/* the collection variant (compute_unit<true> + write_text): rewritten bytes (out_bytes, 16-byte aligned) and their offsets,
 * the tuple stream of the rewritten documents.  Large documents: rewritten on the host, lexed by the large path's replay. */
extern "C" uint64_t hs_warp_collection_batch(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, uint8_t *out_bytes, uint64_t *out_doc_off,
                                             obm_tuple *out, uint64_t cap, uint64_t *tuple_off, uint64_t *stats) {
    using namespace obmw;
    static WarpSmem S; static wemu::Warp W; static bool poisoned = false;
    if (!poisoned) { memset(&S, 0x2B, sizeof S); poisoned = true; }
    const uint64_t total = doc_off[ndocs];
    const uint64_t ntiles = total / TILE + 1;
    std::vector<uint32_t> counts(ndocs + 1, 0);
    std::vector<uint64_t> lg_off(ndocs + 1, 0);
    std::vector<std::vector<uint8_t>> lg_text(ndocs);
    for (uint32_t d = 0; d < ndocs; d++) {
        const uint32_t n = (uint32_t)(doc_off[d + 1] - doc_off[d]);
        if (n > MAXDOC) lg_text[d] = host_rewrite(bytes + doc_off[d], n);
        lg_off[d + 1] = lg_off[d] + lg_text[d].size();
    }
    uint32_t status[4] = {0, 0, 0, 0}; unsigned long long totals[2] = {0, 0};
    WArgs A; memset(&A, 0, sizeof A);
    A.bytes = bytes; A.doc_off = doc_off; A.ndocs = ndocs; A.total_bytes = total; A.ntiles = (uint32_t)ntiles;
    A.counts = counts.data(); A.out = out; A.out_cap = cap; A.tuple_off = tuple_off; A.status = status; A.totals = totals;
    A.lg_off = lg_off.data(); A.out_bytes = out_bytes; A.out_doc_off = out_doc_off;
    std::vector<WRec> recs(ntiles); std::vector<uint64_t> ubase(ntiles + 1, 0);
    uint32_t d = 0;
    for (uint64_t t = 0; t < ntiles; t++) {
        const uint32_t d0 = d;
        while (d < ndocs && doc_off[d] < (t + 1) * (uint64_t)TILE) d++;
        recs[t] = make_wrec(doc_off, d0, d);
        ubase[t + 1] = ubase[t] + recs[t].n_units;
    }
    const uint32_t nunits = (uint32_t)ubase[ntiles];
    std::vector<uint64_t> unit_bytes;
    HostHooks H; H.bytes_of_unit = &unit_bytes;
    uint64_t st_m = 0, st_l = 0, st_e = 0, st_f = 0, chain = 0, bchain = 0;
    UnitRegs pend[32]; uint64_t pend_base = 0; bool have_pend = false;
    std::vector<uint32_t> large_docs;
    auto add_acc = [&](WAcc *a) { for (int l = 0; l < 32; l++) { st_m += a[l].markers; st_l += a[l].lexemes; st_e += a[l].exact; st_f += a[l].fatal; } };
    for (uint64_t t = 0; t < ntiles; t++) {
        for (uint32_t k = 0; k < recs[t].n_units; k++) {
            uint32_t da, db, extra;
            wrec_unit(recs[t], k, da, db, extra);
            if (extra) {
                const uint32_t dl = db;
                obm::SmallSink s(nullptr, 0); obm::Lexer<obm::SmallSink> lx(TBL, lg_text[dl].data(), (uint32_t)lg_text[dl].size(), s);
                int st = lx.run<false>(); counts[dl] = s.n_tuples; st_m += s.n_markers; st_l += s.n_lexemes; st_e++; st_f += st == obm::RUN_FATAL;
                large_docs.push_back(dl);
            }
            const uint32_t u = (uint32_t)ubase[t] + k;
            UnitRegs R[32];
            const UnitDesc D = make_desc(A, u, da, db, extra);
            wemu::run(W, [&]() { compute_unit<true>(S, S.set, A, TBL, H, D, false, R[wemu::lane()]); });
            if (unit_bytes.size() <= u || unit_bytes[u] != R[0].nbytes) { fprintf(stderr, "hostsim: unit %u published no / another byte count\n", u); abort(); }
            const uint64_t my_base = chain; chain += R[0].total;
            const uint64_t my_bbase = bchain; bchain += R[0].nbytes;
            wemu::run(W, [&]() { write_text(S, A, R[wemu::lane()], my_bbase); });
            if (have_pend) { wemu::run(W, [&]() { write_fin(S, A, pend[wemu::lane()], nunits, pend_base); }); have_pend = false; }
            WAcc a[32]; memset(a, 0, sizeof a);
            bool deferred[32]; memset(deferred, 0, sizeof deferred);
            if (!R[0].needs_text) wemu::run(W, [&]() { deferred[wemu::lane()] = assemble_fin(S, S.set, R[wemu::lane()], a[wemu::lane()]); });
            if (deferred[0]) { memcpy(pend, R, sizeof R); pend_base = my_base; have_pend = true; }
            else wemu::run(W, [&]() { write_unit(S, S.set, A, TBL, R[wemu::lane()], nunits, my_base, a[wemu::lane()]); });
            add_acc(a);
        }
    }
    if (have_pend) wemu::run(W, [&]() { write_fin(S, A, pend[wemu::lane()], nunits, pend_base); });
    for (uint32_t dl : large_docs) {
        const uint64_t at = tuple_off[dl];
        obm::WriteSink sink(out + at, at < cap ? cap - at : 0);
        obm::Lexer<obm::WriteSink> lx(TBL, lg_text[dl].data(), (uint32_t)lg_text[dl].size(), sink);
        lx.run<false>();
        if (out_doc_off[dl + 1] - out_doc_off[dl] != lg_text[dl].size()) { fprintf(stderr, "hostsim: large document %u misplaced\n", dl); abort(); }
        if (!lg_text[dl].empty()) memcpy(out_bytes + out_doc_off[dl], lg_text[dl].data(), lg_text[dl].size());
    }
    if (ndocs == 0) { tuple_off[0] = 0; out_doc_off[0] = 0; }
    if (stats) { stats[0] = st_m; stats[1] = st_l; stats[2] = st_e; stats[3] = st_f; }
    return chain;
}
