/* Host build of the fused warp kernel's unit descriptors (csrc/obm_warp.h, obm_warp_core.h), for tests/test_unit_desc.py:
 * the tiles' records as k_wtile_index / k_wunits make them, the descriptor table as k_wunit_descs writes it, and, for every
 * unit, what the scan makes of its descriptor against what the tile record says directly. */
#include <cstdint>
#include <cstring>
#include <vector>
struct uint4 { uint32_t x, y, z, w; };
#define WLANE() 0u
#define WBALLOT(p) ((p) ? 1u : 0u)
#define WSHFL(v, s) (v)
#define WSHFL_UP(v, d) (v)
#define WSYNC()
#define WTEXT(S) ((const uint8_t *)(S).text)
#define WATOMIC_OR(p, v) (*(p) |= (v))
#include "../operator-builder_b200/csrc/obm_warp_core.h"

/* per unit, 7 words {u, da, db, extra, skew, span, base_abs}: got = make_desc over the descriptor table, want = wrec_unit and the
 * unit's two document offsets read directly.  Returns the number of units (at most cap are written). */
extern "C" uint64_t ud_descs(const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, uint64_t *got, uint64_t *want, uint64_t cap) {
    using namespace obmw;
    const uint64_t ntiles = doc_off[ndocs] / TILE + 1;
    std::vector<WRec> recs(ntiles);
    std::vector<uint64_t> ubase(ntiles + 1, 0);
    uint32_t d = 0;
    for (uint64_t t = 0; t < ntiles; t++) {
        const uint32_t d0 = d;
        while (d < ndocs && doc_off[d] < (t + 1) * (uint64_t)TILE) d++;
        recs[t] = make_wrec(doc_off, d0, d);
        ubase[t + 1] = ubase[t] + recs[t].n_units;
    }
    std::vector<WUnit> units(ubase[ntiles]);
    for (uint64_t t = 0; t < ntiles; t++)
        for (uint32_t k = 0; k < recs[t].n_units; k++) units[ubase[t] + k] = make_wunit(doc_off, recs[t], k);
    WArgs A;
    memset(&A, 0, sizeof A);
    A.bytes = bytes; A.doc_off = doc_off; A.ndocs = ndocs;
    const uint64_t base = (uint64_t)(uintptr_t)bytes;
    for (uint64_t t = 0; t < ntiles; t++) {
        for (uint32_t k = 0; k < recs[t].n_units; k++) {
            const uint64_t u = ubase[t] + k;
            if (u >= cap) continue;
            const UnitDesc D = make_desc(A, (uint32_t)u, units[u]);
            const uint64_t g[7] = {D.u, D.da, D.db, D.extra, D.skew, D.span, D.base_abs};
            uint32_t da, db, extra;
            wrec_unit(recs[t], k, da, db, extra);
            uint64_t skew = 0, span = 0, abs_base = 0;
            if (db > da) {
                const uint64_t abs0 = base + doc_off[da];
                skew = abs0 & 15u; span = doc_off[db] - doc_off[da] + skew; abs_base = abs0 & ~15ull;
            }
            const uint64_t w[7] = {u, da, db, extra, skew, span, abs_base};
            memcpy(got + 7 * u, g, sizeof g);
            memcpy(want + 7 * u, w, sizeof w);
        }
    }
    return units.size();
}
