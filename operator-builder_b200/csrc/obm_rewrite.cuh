/*
 * obm_rewrite.cuh -- Manifest.LoadContent's collection rewrite (internal/workload/v1/manifests/manifest.go:89-95) as ONE
 * pass over a packed batch: the text is read once and the rewritten text is written once (2 B of traffic per input byte;
 * r01's kernel read it twice, a warp per document, and moved the runs between deletions byte-interleaved).
 *
 *     ReplaceAll(ReplaceAll(content, "+operator-builder:collection:field", "+operator-builder:field"), "collectionField", "field")
 *
 * Both replacements are deletions ("collection:" at +18 of the first pattern; "collection" of the second, whose 'F' is
 * lowered); the patterns cannot overlap each other or themselves and the first replacement cannot create an occurrence of
 * the second (obm_lib.cu, k_rewrite_collection), so the rewrite is a stream compaction of the batch:
 *
 *   a CTA takes CHUNKS of RW_CH bytes of the packed batch by ticket (document boundaries play no part in the staging)
 *   stage     the chunk and a halo of 48 bytes either side -> shared memory (16 bytes per thread and step)
 *   detect    exact SIMD byte tests for the rare anchors '+' and 'F'; candidates are verified byte by byte in shared memory
 *             and must lie inside ONE document (no document offset strictly inside the match: a bisection of doc_off between
 *             the tile index entries around the match) -> match list
 *   apply     deleted-byte bitmap of the chunk (a match that starts in the previous chunk is seen through the halo), 'F' -> 'f'
 *   count     kept bytes per 32-byte word -> exclusive prefix; the chunk total goes through a decoupled look-back over chunks
 *   offsets   new_off[d] = kept bytes before doc_off[d], for the documents that start in the chunk (tile index)
 *   write     OUTPUT-centric: a thread per aligned 16-byte word of the output; its first byte's source position is a rank
 *             query on the bitmap (a bisection over at most deleted/32 + 2 words); when the 16 source bytes are
 *             contiguous (almost always) they are five shared-memory words funnel-shifted into four; the other words (a
 *             deletion inside, or shared with the neighbouring chunk) are collected and then written a thread per byte
 *
 * Requires 16-byte aligned input and output buffers (the caller falls back to k_rewrite_collection otherwise).
 */
#ifndef OBM_REWRITE_CUH
#define OBM_REWRITE_CUH

namespace obmrw {

constexpr uint32_t RW_CH = 12288;          /* bytes per chunk */
constexpr uint32_t RW_HALO = 48;           /* staged either side (a pattern is 34 bytes) */
constexpr uint32_t RW_THREADS = 256;
constexpr uint32_t RW_NW = RW_CH / 32;     /* bitmap words */
constexpr uint32_t RW_MCAP = 1280;         /* matches per chunk: at most 12288/15 + 48/15 of the short pattern */
constexpr uint32_t RW_SLOTS = (RW_CH + 2 * RW_HALO) / 16;

struct RwSmem {
    alignas(16) uint8_t text[RW_CH + 2 * RW_HALO + 16]; /* text[i] = byte c0 - RW_HALO + i */
    uint32_t del[RW_NW + 1];                            /* bit = byte of the chunk is dropped; [RW_NW]: zero */
    uint32_t kpre[RW_NW + 1];                           /* kept bytes in words [0, w) */
    uint32_t mlist[RW_MCAP];                            /* match: (position relative to c0 - RW_HALO) << 1 | second pattern */
    uint32_t rowtot[RW_NW / 32];
    uint32_t nmatch, ticket, kept;
    uint64_t excl;
};

/* first document d with doc_off[d] >= t * RW_CH for t <= nchunks; the table closes with ndocs */
__global__ void __launch_bounds__(256)
k_rw_tile_index(const uint64_t *__restrict__ doc_off, uint32_t ndocs, uint32_t nchunks, uint32_t *__restrict__ tile_first) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d > ndocs) return;
    const uint64_t tprev_plus1 = d == 0 ? 0 : doc_off[d - 1] / RW_CH + 1;
    const uint64_t tcur = d == ndocs ? (uint64_t)nchunks + 1 : doc_off[d] / RW_CH;
    for (uint64_t t = tprev_plus1; t <= tcur && t <= (uint64_t)nchunks + 1; t++) tile_first[t] = d;
}

__device__ __forceinline__ uint32_t rw_eq16(const uint4 &v, uint32_t pat) { /* 16-bit mask of the bytes equal to pat's byte */
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t z[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const uint32_t t = w[k] ^ pat;
        z[k] = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t) & 0x80808080u; /* bit 7 of every zero byte */
    }
    if (!(z[0] | z[1] | z[2] | z[3])) return 0; /* the anchors are rare */
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) m |= ((z[k] * 0x00204081u) >> 28) << (4 * k);
    return m;
}
/* the patterns as little-endian words (the last one padded with zeros and compared under a mask) */
__device__ __forceinline__ constexpr uint32_t rw_w(const char *p, int i, int len) {
    return (i < len ? (uint32_t)(uint8_t)p[i] : 0u) | (i + 1 < len ? (uint32_t)(uint8_t)p[i + 1] << 8 : 0u) |
           (i + 2 < len ? (uint32_t)(uint8_t)p[i + 2] << 16 : 0u) | (i + 3 < len ? (uint32_t)(uint8_t)p[i + 3] << 24 : 0u);
}
template <int LEN>
__device__ __forceinline__ bool rw_verify(const uint32_t *tw, uint32_t i, const char (&pat)[LEN + 1]) {
    const uint32_t wq = i >> 2, s8 = (i & 3u) * 8u;
    uint32_t a = tw[wq];
#pragma unroll
    for (int k = 0; k < LEN; k += 4) {
        const uint32_t b = tw[wq + k / 4 + 1];
        const uint32_t got = __funnelshift_r(a, b, s8);
        const uint32_t mask = LEN - k >= 4 ? 0xFFFFFFFFu : (1u << (8 * (LEN - k))) - 1u;
        if ((got & mask) != rw_w(pat, k, LEN)) return false;
        a = b;
    }
    return true;
}

/* no document offset strictly inside (p, p + len): the match lies in one document */
__device__ __forceinline__ bool rw_one_doc(const uint64_t *__restrict__ doc_off, const uint32_t *__restrict__ tile_first, uint32_t ndocs,
                                           uint32_t nchunks, uint64_t p, uint32_t len) {
    const uint64_t t = p / RW_CH;
    uint32_t lo = tile_first[t];                                            /* every document before it starts below t * RW_CH <= p */
    uint32_t hi = t + 2 <= (uint64_t)nchunks + 1 ? tile_first[t + 2] : ndocs; /* starts at or beyond (t + 2) * RW_CH > p + len, or is the end */
    if (hi > ndocs) hi = ndocs;
    while (lo < hi) { /* first k with doc_off[k] > p */
        const uint32_t mid = (lo + hi) >> 1;
        if (doc_off[mid] > p) hi = mid; else lo = mid + 1;
    }
    return doc_off[lo] >= p + len; /* lo <= ndocs: doc_off[ndocs] = total >= p + len was checked by the caller */
}

/* source position (chunk-relative) of output byte j of the chunk */
__device__ __forceinline__ uint32_t rw_select(const RwSmem &S, uint32_t j, uint32_t dropped) {
    uint32_t lo = j >> 5, hi = (j + dropped) >> 5;
    if (hi > RW_NW - 1) hi = RW_NW - 1;
    while (lo < hi) { /* largest w with kpre[w] <= j */
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (S.kpre[mid] <= j) lo = mid; else hi = mid - 1;
    }
    const uint32_t r = j - S.kpre[lo], keep = ~S.del[lo];
    if (keep == 0xFFFFFFFFu) return (lo << 5) + r;
    uint32_t m = keep, q = r, b = 0, cnt; /* position of the (q+1)-th set bit: five popcount steps */
    cnt = (uint32_t)__popc(m & 0xFFFFu); if (q >= cnt) { q -= cnt; b = 16; m >>= 16; }
    cnt = (uint32_t)__popc(m & 0xFFu);   if (q >= cnt) { q -= cnt; b += 8; m >>= 8; }
    cnt = (uint32_t)__popc(m & 0xFu);    if (q >= cnt) { q -= cnt; b += 4; m >>= 4; }
    cnt = (uint32_t)__popc(m & 0x3u);    if (q >= cnt) { q -= cnt; b += 2; m >>= 2; }
    if (q >= (m & 1u)) b += 1;
    return (lo << 5) + b;
}

template <bool WRITE>
__global__ void __launch_bounds__(RW_THREADS)
k_rw_chunks(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, uint32_t ndocs, uint64_t total, uint32_t nchunks,
            const uint32_t *__restrict__ tile_first, volatile uint64_t *state, uint32_t *ticket, uint64_t *__restrict__ new_off,
            uint8_t *__restrict__ out, uint64_t out_cap) {
    __shared__ RwSmem S;
    const uint32_t tid = threadIdx.x, lane = tid & 31;
    const uint64_t total16 = (total + 15) & ~15ull;
    const uint32_t *tw = reinterpret_cast<const uint32_t *>(S.text);
    for (;;) {
        __syncthreads(); /* the previous chunk's shared memory is dead */
        if (tid == 0) { S.ticket = atomicAdd(ticket, 1u); S.nmatch = 0; }
        for (uint32_t w = tid; w <= RW_NW; w += RW_THREADS) S.del[w] = 0;
        __syncthreads();
        const uint32_t c = S.ticket;
        if (c >= nchunks) return;
        const uint64_t c0 = (uint64_t)c * RW_CH;
        const uint32_t n = total - c0 < RW_CH ? (uint32_t)(total - c0) : RW_CH;
        /* ---- stage ---- */
        for (uint32_t s = tid; s < RW_SLOTS + 1; s += RW_THREADS) {
            const int64_t a = (int64_t)c0 - RW_HALO + 16 * (int64_t)s;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (a >= 0 && (uint64_t)a < total16) v = *reinterpret_cast<const uint4 *>(bytes + a);
            reinterpret_cast<uint4 *>(S.text)[s] = v;
        }
        __syncthreads();
        /* ---- detect ---- */
        for (uint32_t s = tid; s < RW_SLOTS; s += RW_THREADS) {
            const uint4 v = reinterpret_cast<const uint4 *>(S.text)[s];
            uint32_t plus = rw_eq16(v, 0x2B2B2B2Bu), eff = rw_eq16(v, 0x46464646u);
            while (plus | eff) {
                const bool second = plus == 0;
                uint32_t &m = second ? eff : plus;
                const uint32_t b = (uint32_t)__ffs((int)m) - 1u; m &= m - 1u;
                const int32_t i = (int32_t)(16 * s + b) - (second ? 10 : 0); /* match start, relative to c0 - RW_HALO */
                const uint32_t len = second ? 15u : 34u;
                if (i < 0 || i + len > RW_CH + 2 * RW_HALO) continue;
                const int64_t p = (int64_t)c0 - RW_HALO + i;
                if (p < 0 || (uint64_t)p + len > total) continue;
                if (!(second ? rw_verify<15>(tw, (uint32_t)i, "collectionField") : rw_verify<34>(tw, (uint32_t)i, "+operator-builder:collection:field"))) continue;
                /* what this chunk takes from the match: the dropped bytes (and the lowered letter) inside [c0, c0 + n) */
                const int64_t d0 = p + (second ? 0 : 18), d1 = p + (second ? 11 : 29); /* second: the 'F' at d1 - 1 is this chunk's business too */
                if (d1 <= (int64_t)c0 || d0 >= (int64_t)(c0 + n)) continue;
                if (!rw_one_doc(doc_off, tile_first, ndocs, nchunks, (uint64_t)p, len)) continue;
                const uint32_t k = atomicAdd(&S.nmatch, 1u);
                if (k < RW_MCAP) S.mlist[k] = ((uint32_t)i << 1) | (second ? 1u : 0u);
            }
        }
        __syncthreads();
        /* ---- apply ---- */
        const uint32_t nm = S.nmatch < RW_MCAP ? S.nmatch : RW_MCAP;
        for (uint32_t k = tid; k < nm; k += RW_THREADS) {
            const uint32_t e = S.mlist[k], i = e >> 1;
            const bool second = e & 1u;
            const int32_t r0 = (int32_t)i - (int32_t)RW_HALO + (second ? 0 : 18), r1 = r0 + (second ? 10 : 11); /* chunk-relative dropped range */
            for (int32_t r = r0 < 0 ? 0 : r0; r < r1 && r < (int32_t)n; r++) atomicOr(&S.del[r >> 5], 1u << (r & 31));
            if (second && r1 >= 0 && r1 < (int32_t)n) S.text[RW_HALO + r1] = 'f';
        }
        if (tid >= 64 && n < RW_CH) /* the bytes past the end of the batch are not output */
            for (uint32_t r = n + (tid - 64); r < RW_CH; r += RW_THREADS - 64) atomicOr(&S.del[r >> 5], 1u << (r & 31));
        __syncthreads();
        /* ---- count: a warp per 32 words, then the row totals ---- */
        for (uint32_t row = tid >> 5; row < RW_NW / 32; row += RW_THREADS / 32) {
            const uint32_t kq = 32u - (uint32_t)__popc(S.del[row * 32 + lane]);
            uint32_t inc = kq;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if ((int)lane >= o) inc += t; }
            S.kpre[row * 32 + lane] = inc - kq;
            if (lane == 31) S.rowtot[row] = inc;
        }
        __syncthreads();
        {
            uint32_t before = 0, all = 0;
#pragma unroll
            for (uint32_t r = 0; r < RW_NW / 32; r++) { const uint32_t t = S.rowtot[r]; if (r < (tid >> 5)) before += t; if (r < (tid >> 5) + 8) all += t; }
            /* thread tid owns words tid and tid + 256 (rows tid/32 and tid/32 + 8) */
            const uint32_t k0 = S.kpre[tid];
            uint32_t k1 = 0;
            if (tid + RW_THREADS < RW_NW) k1 = S.kpre[tid + RW_THREADS];
            S.kpre[tid] = k0 + before;
            if (tid + RW_THREADS < RW_NW) S.kpre[tid + RW_THREADS] = k1 + all;
        }
        if (tid < 32) {
            uint32_t run = 0;
#pragma unroll
            for (uint32_t r = 0; r < RW_NW / 32; r++) run += S.rowtot[r];
            if (lane == 0) { S.kpre[RW_NW] = run; S.kept = run; }
            /* ---- look-back over the chunks ---- */
            if (lane == 0) { state[c] = (c == 0 ? LB_INCL : LB_AGG) | run; }
            uint64_t sum = 0;
            if (c > 0) {
                int64_t hi = (int64_t)c - 1;
                for (;;) {
                    const int64_t idx = hi - (int64_t)lane;
                    uint64_t s = idx >= 0 ? state[idx] : LB_INCL;
                    const uint32_t pending = __ballot_sync(0xffffffffu, (s >> 62) == 0);
                    const uint32_t incl = __ballot_sync(0xffffffffu, (s >> 62) == 2);
                    const uint32_t upto = incl ? (uint32_t)__ffs((int)incl) - 1u : 31u;
                    const uint32_t need = upto == 31u ? 0xffffffffu : ((2u << upto) - 1u);
                    if (pending & need) { __nanosleep(64); continue; }
                    uint64_t v = lane <= upto ? (s & LB_MASK) : 0;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
                    sum += v;
                    if (incl) break;
                    hi -= 32;
                }
                if (lane == 0) state[c] = LB_INCL | (sum + run);
            }
            if (lane == 0) S.excl = sum;
        }
        __syncthreads();
        const uint64_t E = S.excl;
        const uint32_t K = S.kept;
        /* ---- offsets of the documents that start in the chunk ---- */
        {
            const uint32_t da = tile_first[c], db = tile_first[c + 1];
            for (uint32_t d = da + tid; d < db; d += RW_THREADS) {
                const uint32_t rel = (uint32_t)(doc_off[d] - c0);
                new_off[d] = rel >= RW_CH ? E + K : E + S.kpre[rel >> 5] + (uint32_t)__popc(~S.del[rel >> 5] & ((1u << (rel & 31)) - 1u));
            }
            if (c == nchunks - 1 && tid == 0) new_off[ndocs] = E + K;
        }
        /* ---- write ---- */
        if (WRITE && K) { /* block-uniform */
            const uint32_t dropped = n - K;
            const uint64_t g0 = E >> 4, g1 = (E + K + 15) >> 4;
            if (tid == 0) S.nmatch = 0; /* the match list is dead: it now collects the words that are not one contiguous run */
            __syncthreads();
            for (uint64_t g = g0 + tid; g < g1; g += RW_THREADS) {
                const int64_t j = (int64_t)(g << 4) - (int64_t)E; /* chunk-relative output index of the word's first byte */
                bool fast = j >= 0 && j + 16 <= (int64_t)K && (g << 4) + 16 <= out_cap;
                uint32_t src = 0;
                if (fast) {
                    src = rw_select(S, (uint32_t)j, dropped);
                    const uint32_t w = src >> 5, sh = src & 31;
                    const uint64_t win = (((uint64_t)S.del[w + 1] << 32) | S.del[w]) >> sh; /* w + 1 <= RW_NW: a zero word */
                    fast = (win & 0xFFFFu) == 0 && src + 16 <= n;
                }
                if (fast) {
                    const uint32_t q = RW_HALO + src, wq = q >> 2, s8 = (q & 3u) * 8u;
                    const uint32_t a0 = tw[wq], a1 = tw[wq + 1], a2 = tw[wq + 2], a3 = tw[wq + 3], a4 = tw[wq + 4];
                    uint4 o;
                    o.x = __funnelshift_r(a0, a1, s8); o.y = __funnelshift_r(a1, a2, s8);
                    o.z = __funnelshift_r(a2, a3, s8); o.w = __funnelshift_r(a3, a4, s8);
                    reinterpret_cast<uint4 *>(out)[g] = o;
                } else {
                    S.mlist[atomicAdd(&S.nmatch, 1u)] = (uint32_t)(g - g0); /* at most RW_CH / 16 + 1 <= RW_MCAP words */
                }
            }
            __syncthreads();
            /* the other words (a deletion inside, or shared with a neighbouring chunk), a thread per BYTE */
            const uint32_t nslow = S.nmatch;
            for (uint32_t t = tid; t < nslow * 16u; t += RW_THREADS) {
                const uint64_t o = ((g0 + S.mlist[t >> 4]) << 4) + (t & 15u);
                const int64_t jk = (int64_t)o - (int64_t)E;
                if (jk < 0 || jk >= (int64_t)K || o >= out_cap) continue;
                out[o] = S.text[RW_HALO + rw_select(S, (uint32_t)jk, dropped)];
            }
        }
    }
}

} // namespace obmrw
#endif
