/*
 * obm_warp.cuh -- device side of the fused warp kernel (logic: obm_warp.h / obm_warp_core.h).
 *
 *   k_wtile_index   tile -> first document starting in it; list of large documents (> obmw::MAXDOC)
 *   k_wunits        per tile: unit count + record; an exclusive scan gives every unit a static id in document order
 *   k_wunit_descs   unit -> 16-byte descriptor (documents, span and byte offset of its text)
 *   k_warp_scan     persistent warps (no block barrier anywhere): a warp takes a unit by ticket, stages the text of
 *                   each of its units with one TMA bulk copy (cp.async.bulk + mbarrier) into its own slice of shared
 *                   memory and runs obmw::process_unit on it
 */
#pragma once
#include "obm_fast.cuh"
#include "obm_pipe.cuh"

#define WLANE() (threadIdx.x & 31u)
#define WBALLOT(p) __ballot_sync(0xffffffffu, (p))
#define WSHFL(v, s) __shfl_sync(0xffffffffu, (v), (s))
#define WSHFL_UP(v, d) __shfl_up_sync(0xffffffffu, (v), (d))
#define WSYNC() __syncwarp()
#define WTEXT(S) obm::ShBytes{obmf::smem_u32((S).text), (S).text}
#define WATOMIC_OR(p, v) atomicOr((p), (v))
#define OBMW_FIN_GLOBAL /* W.fin is a slot in global memory: see WarpSmem */
#include "obm_warp_core.h"

#ifndef OBMW_WPC
#define OBMW_WPC 11
#endif

namespace obmw {

constexpr uint32_t WPC = OBMW_WPC; /* warps per CTA; each works alone on its own shared-memory slice and never meets the others (no barrier).  11 =
                                    * every warp the SM's 227 KB of shared memory holds (20.4 KB each, fin in global memory), as ONE CTA so that the
                                    * CTA's warps are dealt round-robin to the SM's four schedulers (single-warp CTAs are not) */
constexpr uint32_t MAX_CTAS = 256; /* grid cap of k_warp_scan (>= the SM count of any H100): the call's scratch holds this many CTAs' fin slots
                                    * without depending on the device it runs on */
enum { WC_TICKET = 0 };
#ifdef OBMW_PHASE_CLOCKS
__device__ unsigned long long g_phase_cycles[PC_N + 1]; /* cycles per bucket summed over warps; [PC_N]: units */
#endif

__global__ void __launch_bounds__(256)
k_wtile_index(const uint64_t *__restrict__ doc_off, uint32_t ndocs, uint32_t ntiles, uint32_t *__restrict__ tile_first,
              uint32_t *__restrict__ large_list, uint32_t *__restrict__ n_large) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d > ndocs) return;
    /* tiles t with  off[d-1] < t*TILE <= off[d]  have tile_first[t] = d; d == ndocs closes the table */
    const uint64_t tprev_plus1 = d == 0 ? 0 : doc_off[d - 1] / TILE + 1;
    const uint64_t tcur = d == ndocs ? (uint64_t)ntiles : doc_off[d] / TILE;
    if (d == ndocs && ndocs > 0 && tprev_plus1 > tcur) return;
    for (uint64_t t = tprev_plus1; t <= tcur && t <= ntiles; t++) tile_first[t] = d;
    if (d < ndocs && doc_off[d + 1] - doc_off[d] > MAXDOC) large_list[atomicAdd(n_large, 1u)] = d;
}

/* unit -> descriptor, after the scan of the unit counts */
__global__ void __launch_bounds__(256)
k_wunit_descs(const uint64_t *__restrict__ doc_off, const WRec *__restrict__ wrec, const uint64_t *__restrict__ ubase, uint32_t ntiles,
              uint64_t units_max, WUnit *__restrict__ units) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    const WRec r = wrec[t];
    const uint64_t u0 = ubase[t];
    for (uint32_t k = 0; k < r.n_units && u0 + k < units_max; k++) units[u0 + k] = make_wunit(doc_off, r, k);
}

__global__ void __launch_bounds__(256)
k_wunits(const uint64_t *__restrict__ doc_off, const uint32_t *__restrict__ tile_first, uint32_t ntiles, uint32_t *__restrict__ nunits, WRec *__restrict__ wrec) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= ntiles) return;
    const WRec r = make_wrec(doc_off, tile_first[t], tile_first[t + 1]);
    nunits[t] = r.n_units;
    wrec[t] = r;
}

struct DevHooks {
    uint32_t phase;
    __device__ __forceinline__ void stage(WarpSmem &S, const void *gsrc, uint32_t nbytes) {
        if (WLANE() == 0 && nbytes) {
            obmf::fence_proxy_async(); /* the warp's earlier generic-proxy accesses to S.text precede the async write */
            obmf::mbar_expect_tx(&S.mbar, nbytes);
            obmf::tma_bulk_g2s(S.text, gsrc, nbytes, &S.mbar);
        }
    }
    __device__ __forceinline__ void stage_wait(WarpSmem &S, uint32_t nbytes) {
        if (nbytes) { obmf::mbar_wait(&S.mbar, phase); phase ^= 1u; }
    }
};

/* ---- the chain over the units' tuple counts ---------------------------------------------------------------
 * Two levels, both fed at PUBLISH time so that nothing on it depends on another warp's (deferred) resolve:
 *   st0[u]   LB_AGG | tuples of unit u                                  (plain store: flag and value are one word)
 *   blk[b]   atomic accumulator of block b = units [32b, 32b+32): count << 56 | sum of tuples
 *   bex[b]   BEX_FLAG | exclusive prefix of block b, stored by whichever unit of the block resolves it first
 * resolve(u) = bex[b] (or a walk back over complete blocks, 32 per step, down to the nearest stored prefix) + the
 * st0 entries of the earlier units of u's own block. */
#define BEX_FLAG (1ull << 63)
__device__ __forceinline__ void chain_publish(uint64_t *st_units, uint64_t *st_blocks, uint32_t u, uint64_t total) {
    if ((threadIdx.x & 31) == 0) {
        reinterpret_cast<volatile uint64_t *>(st_units)[u] = LB_AGG | total;
        atomicAdd(reinterpret_cast<unsigned long long *>(st_blocks) + (u >> 5), (unsigned long long)((1ull << 56) | total));
    }
}
__device__ __forceinline__ uint64_t chain_resolve(uint64_t *st_units, uint64_t *st_blocks, uint32_t u, uint32_t nblocks) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t b = u >> 5, r = u & 31;
    volatile uint64_t *st0 = st_units, *blk = st_blocks, *bex = st_blocks + nblocks;
    uint64_t s, mine;
    uint32_t backoff = 32; /* ns; doubles up to ~2 us: a thousand warps polling at a fixed short interval saturate L2 and slow the
                            * very warps they wait for (marker-dense units resolve right after publishing) */
    for (;;) { /* the block's prefix is read in the same round trip as its st0 entries: once flagged, it never changes */
        s = lane < r ? st0[(b << 5) + lane] : LB_AGG;
        mine = b ? bex[b] : BEX_FLAG;
        if (__ballot_sync(0xffffffffu, (s >> 62) == 0) == 0) break;
        __nanosleep(backoff); if (backoff < 2048) backoff <<= 1;
    }
    uint64_t partial = s & LB_MASK;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) partial += __shfl_xor_sync(0xffffffffu, partial, o);
    uint64_t P = 0;
    if (mine & BEX_FLAG) P = mine & ~BEX_FLAG;
    else {
        int64_t hi = (int64_t)b - 1; /* nearest block not yet accounted for */
        for (;;) {
            const int64_t j = hi - (int64_t)lane;
            const uint64_t e = j > 0 ? bex[j] : BEX_FLAG /* block 0 (and the virtual ones before it) start at 0 */;
            const uint64_t a = j >= 0 ? blk[j] : (32ull << 56);
            const uint32_t have = __ballot_sync(0xffffffffu, (e & BEX_FLAG) != 0);
            const uint32_t part = __ballot_sync(0xffffffffu, (a >> 56) != 32u); /* every block before b is a full one */
            const uint32_t upto = have ? (uint32_t)__ffs((int)have) - 1u : 31u;
            const uint32_t need = upto == 31u ? 0xffffffffu : ((2u << upto) - 1u);
            if (part & need) { __nanosleep(backoff); if (backoff < 2048) backoff <<= 1; continue; }
            uint64_t v = lane <= upto ? (a & ((1ull << 56) - 1)) : 0;
            if (have && lane == upto) v += e & ~BEX_FLAG;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            P += v;
            if (have) break;
            hi -= 32;
        }
        if (lane == 0) bex[b] = BEX_FLAG | P;
    }
    return P + partial;
}

/* Software pipeline over the warp's units: scan unit i (compute_unit), publish its tuple count to the chain, THEN
 * write unit i-1 from W.fin (its exclusive prefix has had a whole unit's time to arrive: no waiting on the chain),
 * assemble unit i into W.fin, scan unit i+1 ...  A unit whose write needs the staged text (documents for the exact
 * lexer, marker lines that are not staged) or that does not fit W.fin is written at once instead. */
__global__ void __launch_bounds__(WPC * 32, 1) /* one CTA per SM: ptxas may take the registers it wants (up to 184 at 11 warps; without the hint it settles for fewer and spills) */
k_warp_scan(WArgs A) {
    extern __shared__ __align__(16) uint8_t smem_raw[];
    WarpSmem &S = reinterpret_cast<WarpSmem *>(smem_raw)[threadIdx.x >> 5];
    const uint32_t lane = threadIdx.x & 31u;
    if (lane == 0) {
        obmf::mbar_init(&S.mbar, 1); obmf::fence_mbar_init();
        S.fin = A.fin_slots + (size_t)(blockIdx.x * WPC + (threadIdx.x >> 5)) * FIN_CAP; /* the warp's own slot (grid <= MAX_CTAS) */
    }
    __syncwarp();
    const obm::Tables T = obmq::dev_tables();
    const uint32_t nunits = (uint32_t)A.ubase[A.ntiles];
    const uint32_t nblocks = (uint32_t)(A.units_max / 32 + 2); /* layout of st_blocks: blk[nblocks] | bex[nblocks] */
    DevHooks H{0};
    WAcc acc{0, 0, 0, 0};
    UnitRegs pend; bool have_pend = false;
    /* unit iterator: UNITS by ticket, in document order (not tiles: a warp that held two units of one tile would publish
     * the second only after writing the first, and with units that resolve right after publishing that serialises the
     * whole chain).  The ticket after next is taken while this unit is processed, and the NEXT unit's descriptor
     * (one 16-byte load) is requested before this unit is scanned, so that it arrives under the scan */
    uint32_t tn = 0;
    auto take_unit = [&](uint32_t &u, WUnit &w) {
        u = __shfl_sync(0xffffffffu, tn, 0);
        if (u >= nunits) return;
        if (lane == 0) tn = atomicAdd(&A.ctl[WC_TICKET], 1u);
        w = A.units[u];
    };
    auto unit_desc = [&](uint32_t u, const WUnit &w) -> UnitDesc {
        if (u >= nunits) { UnitDesc d{0, 0, 0, 0, 0, 0, 0, false, 0}; return d; }
        return make_desc(A, u, w);
    };
    if (lane == 0) tn = atomicAdd(&A.ctl[WC_TICKET], 1u);
#ifdef OBMW_PHASE_CLOCKS
    PhaseClk pc{};
    pc.t0 = (uint32_t)clock64();
    uint32_t pc_units = 0;
#endif
    uint32_t un = 0; WUnit wn{0, 0, 0};
    take_unit(un, wn);
    UnitDesc cur = unit_desc(un, wn);
    bool prestaged = false;
    while (cur.valid) {
        take_unit(un, wn);
        OBMW_PC_MARK(PC_OTHER);
        UnitRegs R;
        compute_unit(S, S.set, A, T, H, cur, prestaged, R OBMW_PC_ARG);
        chain_publish(A.st_tuples, A.st_blocks, R.u, R.total);
        UnitDesc nxt = unit_desc(un, wn);
        prestaged = false;
        /* the staged text is dead unless this unit's write needs it: bring in the next unit's text, and its document offsets, under the
         * assembly and the writes */
        if (prestage_next(R, nxt)) {
            H.stage(S, (const void *)(uintptr_t)nxt.base_abs, desc_load(nxt));
            if (lane <= nxt.db - nxt.da) nxt.doff = A.doc_off[nxt.da + lane];
            prestaged = true;
        }
        OBMW_PC_MARK(PC_OTHER);
        if (have_pend) {
            FinRegs F;
            fin_load(S, A, pend, F); /* the slot's round trip overlaps the chain's */
            const uint64_t base = chain_resolve(A.st_tuples, A.st_blocks, pend.u, nblocks);
            OBMW_PC_MARK(PC_CHAIN);
            write_fin(A, pend, nunits, base, F);
            OBMW_PC_MARK(PC_WRITE);
            have_pend = false;
        }
        if (!R.needs_text && assemble_fin(S, S.set, R, acc)) { pend = R; have_pend = true; OBMW_PC_MARK(PC_AFIN); }
        else {
            OBMW_PC_MARK(PC_AFIN);
            const uint64_t base = chain_resolve(A.st_tuples, A.st_blocks, R.u, nblocks);
            OBMW_PC_MARK(PC_CHAIN);
            write_unit(S, S.set, A, T, R, nunits, base, acc OBMW_PC_ARG);
            OBMW_PC_MARK(PC_WRITE);
        }
        cur = nxt;
#ifdef OBMW_PHASE_CLOCKS
        pc_units++;
#endif
    }
    if (have_pend) {
        FinRegs F;
        fin_load(S, A, pend, F);
        const uint64_t base = chain_resolve(A.st_tuples, A.st_blocks, pend.u, nblocks);
        OBMW_PC_MARK(PC_CHAIN);
        write_fin(A, pend, nunits, base, F);
        OBMW_PC_MARK(PC_WRITE);
    }
#ifdef OBMW_PHASE_CLOCKS
    if (lane == 0) {
#pragma unroll
        for (uint32_t b = 0; b < PC_N; b++) atomicAdd(&g_phase_cycles[b], (unsigned long long)pc.c[b]);
        atomicAdd(&g_phase_cycles[PC_N], (unsigned long long)pc_units);
    }
#endif
    uint32_t markers = acc.markers, lexemes = acc.lexemes, exact = acc.exact, fatal = acc.fatal;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        markers += __shfl_down_sync(0xffffffffu, markers, o); lexemes += __shfl_down_sync(0xffffffffu, lexemes, o);
        exact += __shfl_down_sync(0xffffffffu, exact, o); fatal += __shfl_down_sync(0xffffffffu, fatal, o);
    }
    if (lane == 0) {
        if (markers) atomicAdd(&A.totals[0], (unsigned long long)markers);
        if (lexemes) atomicAdd(&A.totals[1], (unsigned long long)lexemes);
        if (exact) atomicAdd(&A.status[1], exact);
        if (fatal) atomicAdd(&A.status[2], fatal);
    }
}

} /* namespace obmw */
