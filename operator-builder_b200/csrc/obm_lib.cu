/*
 * obm_lib.cu -- libobmarkers.so: CUDA kernels (sm_90a) + the C ABI of include/obmarkers.h.
 *
 * Replaces, for a whole batch of manifests at once, the per-document
 *     lexer.NewLexer(r) ; go l.Run() ; for { l.NextLexeme() }      (internal/markers/lexer/lexer.go:27-53)
 * that internal/markers/parser/parser.go:35,47 starts once per YAML node
 * (internal/markers/inspect/yaml.go:94), driven per manifest by
 * internal/workload/v1/kinds/workload.go:224-285.
 *
 * Kernels in this file
 *   k_exact_count / k_exact_fill   exact path: one thread per document runs obm::Lexer (obm_core.h);
 *                                  handles every input (non-ASCII, invalid UTF-8, multi-line
 *                                  literals, fatal errors, documents of any size)
 *   k_scan_*                       exclusive prefix sum of per-document tuple counts -> doc_tuple_off
 *   k_generate_corpus              synthetic manifests generated in HBM (obm_corpus.h)
 * The fast path (k_tile_scan, obm_fast.cuh) is layered on top of the same core; see DESIGN.md.
 *
 * There is no CPU fallback: without a CUDA device every lexing entry point returns OBM_E_NO_DEVICE.
 */
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>
#include <type_traits>

#include "../../include/obmarkers.h"
#include "go_unicode_tables.h"
#include "obm_core.h"
#include "obm_corpus.h"

extern "C" uint32_t obm_registry_names(const obm_registry *r, const char **names, uint32_t *lens, uint32_t cap);

/* ------------------------------------------------------------------------------------------- */
/* device constants                                                                             */
/* ------------------------------------------------------------------------------------------- */
__device__ const char D_F64_OVERFLOW_DIGITS[] = GO_F64_OVERFLOW_DIGITS;

__device__ __forceinline__ obm::Tables device_tables() {
    obm::Tables T;
    T.letter = D_GO_LETTER_RANGES; T.n_letter = D_GO_LETTER_RANGES_N;
    T.number = D_GO_NUMBER_RANGES; T.n_number = D_GO_NUMBER_RANGES_N;
    T.f64_overflow_digits = D_F64_OVERFLOW_DIGITS;
    return T;
}

/* status words (device uint32[4]) */
enum { ST_OVERFLOW = 0, ST_DOCS_EXACT = 1, ST_DOCS_FATAL = 2, ST_RESERVED = 3 };

#include "obm_fast.cuh"
#include "obm_pipe.cuh"
#include "obm_warp.cuh"
#include "obm_large.h"
static_assert(obmw::MAXDOC > 8192 && obmt::MAXDOC > 8192, "obm_fast_max_large");

/* ------------------------------------------------------------------------------------------- */
/* exact path: one thread per document                                                          */
/* ------------------------------------------------------------------------------------------- */
/* doc_list == nullptr: documents [0, ndocs); otherwise the ids in doc_list[0..ndocs). */
__global__ void __launch_bounds__(128)
k_exact_count(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, const uint32_t *__restrict__ doc_list,
              uint32_t ndocs, const uint32_t *__restrict__ ndocs_dev, uint32_t *__restrict__ counts,
              unsigned long long *__restrict__ totals /* {markers, lexemes} */, uint32_t *__restrict__ status) {
    if (ndocs_dev) ndocs = *ndocs_dev; /* list length decided on the device (large documents) */
    if (blockIdx.x * blockDim.x >= ndocs) return;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t markers = 0, lexemes = 0, fatal = 0;
    if (i < ndocs) {
        uint32_t d = doc_list ? doc_list[i] : i;
        uint64_t o0 = doc_off[d], o1 = doc_off[d + 1];
        obm::Tables T = device_tables();
        obm::CountSink sink;
        obm::Lexer<obm::CountSink> lx(T, bytes + o0, (uint32_t)(o1 - o0), sink);
        int st = lx.run<false>();
        counts[d] = (uint32_t)sink.n_tuples;
        markers = sink.n_markers; lexemes = sink.n_lexemes; fatal = (st == obm::RUN_FATAL);
    }
    /* block-level reduction of the counters, one atomic per block */
    __shared__ uint32_t sm[3];
    if (threadIdx.x < 3) sm[threadIdx.x] = 0;
    __syncthreads();
    for (int o = 16; o > 0; o >>= 1) {
        markers += __shfl_down_sync(0xffffffffu, markers, o);
        lexemes += __shfl_down_sync(0xffffffffu, lexemes, o);
        fatal += __shfl_down_sync(0xffffffffu, fatal, o);
    }
    if ((threadIdx.x & 31) == 0) { atomicAdd(&sm[0], markers); atomicAdd(&sm[1], lexemes); atomicAdd(&sm[2], fatal); }
    __syncthreads();
    if (threadIdx.x == 0) {
        if (totals) { atomicAdd(&totals[0], (unsigned long long)sm[0]); atomicAdd(&totals[1], (unsigned long long)sm[1]); }
        if (status) {
            if (sm[2]) atomicAdd(&status[ST_DOCS_FATAL], sm[2]);
            uint32_t first = blockIdx.x * blockDim.x;
            atomicAdd(&status[ST_DOCS_EXACT], min(blockDim.x, ndocs - first));
        }
    }
}

__global__ void __launch_bounds__(128)
k_exact_fill(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, const uint32_t *__restrict__ doc_list,
             uint32_t ndocs, const uint32_t *__restrict__ ndocs_dev, const uint64_t *__restrict__ tuple_off,
             obm_tuple *__restrict__ out, uint64_t out_cap) {
    if (ndocs_dev) ndocs = *ndocs_dev;
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= ndocs) return;
    uint32_t d = doc_list ? doc_list[i] : i;
    uint64_t o0 = doc_off[d], o1 = doc_off[d + 1];
    uint64_t t0 = tuple_off[d];
    uint64_t room = t0 < out_cap ? out_cap - t0 : 0;
    obm::Tables T = device_tables();
    obm::WriteSink sink(out + t0, room);
    obm::Lexer<obm::WriteSink> lx(T, bytes + o0, (uint32_t)(o1 - o0), sink);
    lx.run<false>();
}

/* ------------------------------------------------------------------------------------------- */
/* exclusive scan u32 counts -> u64 offsets (three small kernels; 8-12 B/doc of traffic)        */
/* ------------------------------------------------------------------------------------------- */
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 8;
constexpr int SCAN_TILE = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ uint64_t block_exclusive_scan(uint64_t v, uint64_t *total) {
    __shared__ uint64_t warp_sums[SCAN_THREADS / 32];
    __shared__ uint64_t block_total;
    uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint64_t incl = v;
    for (int o = 1; o < 32; o <<= 1) { uint64_t t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (uint32_t)o) incl += t; }
    if (lane == 31) warp_sums[wid] = incl;
    __syncthreads();
    if (wid == 0) {
        uint64_t w = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0;
        uint64_t wi = w;
        for (int o = 1; o < 32; o <<= 1) { uint64_t t = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= (uint32_t)o) wi += t; }
        if (lane < SCAN_THREADS / 32) warp_sums[lane] = wi - w;
        if (lane == SCAN_THREADS / 32 - 1) block_total = wi;
    }
    __syncthreads();
    uint64_t excl = incl - v + warp_sums[wid];
    *total = block_total;
    __syncthreads();
    return excl;
}

__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_tiles(const uint32_t *__restrict__ counts, uint32_t n, uint64_t *__restrict__ off, uint64_t *__restrict__ tile_sums) {
    uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    uint32_t c[SCAN_ITEMS]; uint64_t sum = 0;
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { c[k] = (base + k < n) ? counts[base + k] : 0; sum += c[k]; }
    uint64_t total; uint64_t excl = block_exclusive_scan(sum, &total);
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) { if (base + k < n) off[base + k] = excl; excl += c[k]; }
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_sums(uint64_t *__restrict__ tile_sums, uint32_t ntiles, uint64_t *__restrict__ grand_total) {
    uint64_t carry = 0;
    for (uint32_t b = 0; b < ntiles; b += SCAN_THREADS) {
        uint32_t i = b + threadIdx.x;
        uint64_t v = i < ntiles ? tile_sums[i] : 0;
        uint64_t total; uint64_t excl = block_exclusive_scan(v, &total);
        if (i < ntiles) tile_sums[i] = carry + excl;
        carry += total;
    }
    if (threadIdx.x == 0) *grand_total = carry;
}
__global__ void __launch_bounds__(SCAN_THREADS)
k_scan_add(uint64_t *__restrict__ off, uint32_t n, const uint64_t *__restrict__ tile_sums, uint64_t out_cap, uint32_t *__restrict__ status) {
    uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
    uint64_t add = tile_sums[blockIdx.x];
#pragma unroll
    for (int k = 0; k < SCAN_ITEMS; k++) if (base + k < n) off[base + k] += add;
    /* off[n] was written by k_scan_sums (grand_total points at it) */
    if (blockIdx.x == 0 && threadIdx.x == 0 && status && off[n] > out_cap) status[ST_OVERFLOW] = 1;
}

/* ------------------------------------------------------------------------------------------- */
/* large documents (> obmt::MAXDOC bytes): chunk-parallel exact lexing, see obm_large.h          */
/* plan (chunks per document, scan) -> prep (chunk starts, newline counts) -> lines (line numbers; */
/* a chunk without a line start takes the next one's) -> count ->                                */
/* resolve (chain check, offsets, or sequential fallback) ... main scan ... -> fill              */
/* ------------------------------------------------------------------------------------------- */
struct LargeWs {
    const uint32_t *large_list; const uint32_t *n_large; uint32_t max_large;
    uint32_t *lch; uint64_t *lbase; uint64_t *lsums; uint32_t *lvalid;
    uint32_t *cs, *cnl, *cline, *ccnt, *cend, *cflag, *cmk, *clx; uint64_t *choff;
};
static uint64_t large_chunks_max(uint64_t total_bytes) { return total_bytes / obml::LCHUNK + obm_fast_max_large(total_bytes) + 2; }
static uint32_t scan_tiles(uint32_t ndocs);
static uint64_t align_up(uint64_t v, uint64_t a);
static uint64_t large_scratch_bytes(uint64_t total_bytes) {
    const uint64_t ml = obm_fast_max_large(total_bytes), nc = large_chunks_max(total_bytes);
    return align_up((ml + 1) * 4, 256) + align_up((ml + 2) * 8, 256) + align_up(((uint64_t)scan_tiles((uint32_t)ml + 1) + 1) * 8, 256) +
           align_up((ml + 1) * 4, 256) + 8 * align_up((nc + 1) * 4, 256) + align_up((nc + 1) * 8, 256);
}
static LargeWs large_carve(void *ws, uint64_t total_bytes, const uint32_t *large_list, const uint32_t *n_large) {
    const uint64_t ml = obm_fast_max_large(total_bytes), nc = large_chunks_max(total_bytes);
    uint8_t *q = (uint8_t *)ws; LargeWs W;
    W.large_list = large_list; W.n_large = n_large; W.max_large = (uint32_t)ml;
    W.lch = (uint32_t *)q; q += align_up((ml + 1) * 4, 256);
    W.lbase = (uint64_t *)q; q += align_up((ml + 2) * 8, 256);
    W.lsums = (uint64_t *)q; q += align_up(((uint64_t)scan_tiles((uint32_t)ml + 1) + 1) * 8, 256);
    W.lvalid = (uint32_t *)q; q += align_up((ml + 1) * 4, 256);
    uint32_t **arr[8] = {&W.cs, &W.cnl, &W.cline, &W.ccnt, &W.cend, &W.cflag, &W.cmk, &W.clx};
    for (auto a : arr) { *a = (uint32_t *)q; q += align_up((nc + 1) * 4, 256); }
    W.choff = (uint64_t *)q;
    return W;
}
/* the large document that owns global chunk g: last i with lbase[i] <= g */
__device__ __forceinline__ uint32_t large_of_chunk(const LargeWs &W, uint32_t n_large, uint64_t g) {
    uint32_t lo = 0, hi = n_large;
    while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (W.lbase[mid] <= g) lo = mid; else hi = mid; }
    return lo;
}
__global__ void __launch_bounds__(256)
k_large_nchunks(const uint64_t *__restrict__ doc_off, LargeWs W) {
    const uint32_t n_large = *W.n_large;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= W.max_large; i += gridDim.x * blockDim.x) {
        uint32_t v = 0;
        if (i < n_large) { const uint32_t d = W.large_list[i]; v = obml::n_chunks((uint32_t)(doc_off[d + 1] - doc_off[d])); }
        W.lch[i] = v;
    }
}
__global__ void __launch_bounds__(128)
k_large_prep(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, LargeWs W) {
    const uint32_t n_large = *W.n_large;
    if (n_large == 0) return;
    const uint64_t total = W.lbase[W.max_large + 1];
    for (uint64_t g = blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t i = large_of_chunk(W, n_large, g), d = W.large_list[i], c = (uint32_t)(g - W.lbase[i]);
        const uint8_t *doc = bytes + doc_off[d]; const uint32_t n = (uint32_t)(doc_off[d + 1] - doc_off[d]);
        uint32_t sk;
        W.cs[g] = obml::chunk_start(doc, n, c, &sk);
        W.cline[g] = sk;
        W.cnl[g] = obml::chunk_newlines(doc, n, c) | (obml::chunk_non_ascii(doc, n, c) ? 0x80000000u : 0u);
    }
}
__global__ void __launch_bounds__(128)
k_large_lines(LargeWs W) {
    const uint32_t n_large = *W.n_large;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_large; i += gridDim.x * blockDim.x) {
        const uint64_t g0 = W.lbase[i]; const uint32_t nc = (uint32_t)(W.lbase[i + 1] - g0);
        uint32_t acc = 0, na = 0;
        for (uint32_t c = 0; c < nc; c++) {
            const uint32_t sk = W.cline[g0 + c], v = W.cnl[g0 + c];
            W.cline[g0 + c] = 1u + acc + sk; acc += v & 0x7FFFFFFFu; na |= v >> 31;
        }
        obml::resolve_chunk_starts(W.cs + g0, W.cline + g0, nc);
        W.lch[i] = na ? 0u : 1u; /* reused after the scan: 1 = the document is all ASCII (fast lexer instantiation) */
    }
}
__global__ void __launch_bounds__(128)
k_large_count(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, LargeWs W) {
    const uint32_t n_large = *W.n_large;
    if (n_large == 0) return;
    const uint64_t total = W.lbase[W.max_large + 1];
    const obm::Tables T = device_tables();
    for (uint64_t g = blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t i = large_of_chunk(W, n_large, g), d = W.large_list[i], c = (uint32_t)(g - W.lbase[i]);
        const uint32_t nc = (uint32_t)(W.lbase[i + 1] - W.lbase[i]);
        const uint8_t *doc = bytes + doc_off[d]; const uint32_t n = (uint32_t)(doc_off[d + 1] - doc_off[d]);
        const uint32_t stop = c + 1 < nc ? W.cs[g + 1] : n;
        obm::SmallSink sink(nullptr, 0);
        uint32_t end;
        W.cflag[g] = W.lch[i] ? obml::lex_chunk<obm::SmallSink, true>(T, doc, n, W.cs[g], W.cline[g], stop, sink, &end)
                              : obml::lex_chunk<obm::SmallSink, false>(T, doc, n, W.cs[g], W.cline[g], stop, sink, &end);
        W.cend[g] = end; W.ccnt[g] = sink.n_tuples; W.cmk[g] = sink.n_markers; W.clx[g] = sink.n_lexemes;
    }
}
__global__ void __launch_bounds__(128)
k_large_resolve(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, LargeWs W, uint32_t *__restrict__ counts,
                unsigned long long *__restrict__ totals, uint32_t *__restrict__ status) {
    const uint32_t n_large = *W.n_large;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n_large; i += gridDim.x * blockDim.x) {
        const uint32_t d = W.large_list[i];
        const uint64_t g0 = W.lbase[i]; const uint32_t nc = (uint32_t)(W.lbase[i + 1] - g0);
        const uint32_t n = (uint32_t)(doc_off[d + 1] - doc_off[d]);
        bool valid = true;
        for (uint32_t c = 0; c < nc; c++) {
            const uint32_t stop = c + 1 < nc ? W.cs[g0 + c + 1] : n;
            if (W.cflag[g0 + c] || W.cend[g0 + c] != stop) { valid = false; break; }
        }
        uint64_t mk = 0, lx = 0; uint32_t fatal = 0;
        if (valid) {
            uint64_t off = 0;
            for (uint32_t c = 0; c < nc; c++) { W.choff[g0 + c] = off; off += W.ccnt[g0 + c]; mk += W.cmk[g0 + c]; lx += W.clx[g0 + c]; }
            counts[d] = (uint32_t)(off + 1); lx += 1; /* EOF */
        } else {
            /* a construct crosses a chunk boundary, or the document ends in a fatal error: lex it sequentially */
            const obm::Tables T = device_tables();
            obm::CountSink sink;
            obm::Lexer<obm::CountSink> lex(T, bytes + doc_off[d], n, sink);
            const int st = lex.run<false>();
            counts[d] = (uint32_t)sink.n_tuples; mk = sink.n_markers; lx = sink.n_lexemes; fatal = st == obm::RUN_FATAL;
        }
        W.lvalid[i] = valid ? 1u : 0u;
        if (totals) { atomicAdd(&totals[0], (unsigned long long)mk); atomicAdd(&totals[1], (unsigned long long)lx); }
        if (status) { atomicAdd(&status[ST_DOCS_EXACT], 1u); if (fatal) atomicAdd(&status[ST_DOCS_FATAL], 1u); }
    }
}
__global__ void __launch_bounds__(128)
k_large_fill(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, LargeWs W, const uint64_t *__restrict__ tuple_off,
             obm_tuple *__restrict__ out, uint64_t out_cap) {
    const uint32_t n_large = *W.n_large;
    if (n_large == 0) return;
    const uint64_t total = W.lbase[W.max_large + 1];
    const obm::Tables T = device_tables();
    for (uint64_t g = blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t i = large_of_chunk(W, n_large, g), d = W.large_list[i], c = (uint32_t)(g - W.lbase[i]);
        const uint32_t nc = (uint32_t)(W.lbase[i + 1] - W.lbase[i]);
        const uint8_t *doc = bytes + doc_off[d]; const uint32_t n = (uint32_t)(doc_off[d + 1] - doc_off[d]);
        if (!W.lvalid[i]) {
            if (c == 0) {
                const uint64_t t0 = tuple_off[d];
                obm::WriteSink sink(out + t0, t0 < out_cap ? out_cap - t0 : 0);
                obm::Lexer<obm::WriteSink> lex(T, doc, n, sink);
                lex.run<false>();
            }
            continue;
        }
        const uint64_t t0 = tuple_off[d] + W.choff[g];
        const uint32_t stop = c + 1 < nc ? W.cs[g + 1] : n;
        obm::WriteSink sink(out + t0, t0 < out_cap ? out_cap - t0 : 0);
        uint32_t end;
        if (W.lch[i]) obml::lex_chunk<obm::WriteSink, true>(T, doc, n, W.cs[g], W.cline[g], stop, sink, &end);
        else obml::lex_chunk<obm::WriteSink, false>(T, doc, n, W.cs[g], W.cline[g], stop, sink, &end);
        if (c == nc - 1) { const uint64_t e = t0 + W.ccnt[g]; if (e < out_cap) out[e] = OBM_TUPLE(OBM_K_EOF, n, 0); }
    }
}

static void large_count_launch(cudaStream_t st, int sms, const uint8_t *d_bytes, const uint64_t *d_doc_off, const LargeWs &W,
                               uint32_t *counts, unsigned long long *totals, uint32_t *status) {
    const uint32_t n = W.max_large + 1, nt = scan_tiles(n);
    const uint32_t g = (uint32_t)sms * 8u, gl = (n + 255) / 256 < g ? (n + 255) / 256 : g;
    k_large_nchunks<<<gl, 256, 0, st>>>(d_doc_off, W);
    k_scan_tiles<<<nt, SCAN_THREADS, 0, st>>>(W.lch, n, W.lbase, W.lsums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(W.lsums, nt, W.lbase + n);
    k_scan_add<<<nt, SCAN_THREADS, 0, st>>>(W.lbase, n, W.lsums, ~0ull, nullptr);
    k_large_prep<<<g, 128, 0, st>>>(d_bytes, d_doc_off, W);
    k_large_lines<<<gl, 128, 0, st>>>(W);
    k_large_count<<<g, 128, 0, st>>>(d_bytes, d_doc_off, W);
    k_large_resolve<<<gl, 128, 0, st>>>(d_bytes, d_doc_off, W, counts, totals, status);
}
constexpr uint32_t LARGE_COUNT_LAUNCHES = 8;
static void large_fill_launch(cudaStream_t st, int sms, const uint8_t *d_bytes, const uint64_t *d_doc_off, const LargeWs &W,
                              const uint64_t *toff, obm_tuple *d_out, uint64_t out_cap) {
    k_large_fill<<<(uint32_t)sms * 8u, 128, 0, st>>>(d_bytes, d_doc_off, W, toff, d_out, out_cap);
}

/* ------------------------------------------------------------------------------------------- */
/* synthetic corpus                                                                             */
/* ------------------------------------------------------------------------------------------- */
__global__ void __launch_bounds__(128)
k_generate_corpus(uint8_t *__restrict__ bytes, uint64_t *__restrict__ doc_off, uint32_t ndocs, uint32_t doc_bytes,
                  uint64_t first_doc, int flavour) {
    uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d == 0 && doc_off) doc_off[ndocs] = (uint64_t)ndocs * doc_bytes;
    if (d >= ndocs) return;
    if (doc_off) doc_off[d] = (uint64_t)d * doc_bytes;
    obmc::generate_doc(bytes + (uint64_t)d * doc_bytes, doc_bytes, first_doc + d, flavour);
}

/* ------------------------------------------------------------------------------------------- */
/* handle + error plumbing                                                                      */
/* ------------------------------------------------------------------------------------------- */
struct obm_handle {
    int device;
    cudaStream_t stream;
    cudaEvent_t ev[4];
    cudaStream_t side; cudaEvent_t ev_fork, ev_join; /* large-document bookkeeping runs beside k1_scan */
    char err[512];
    /* scratch kept across calls */
    void *scratch; uint64_t scratch_bytes;
    /* device staging for the host-buffer entry point */
    uint8_t *d_bytes; uint64_t d_bytes_cap;
    uint64_t *d_doc_off; uint64_t d_doc_off_cap; /* elements */
    uint64_t *d_tuple_off; uint64_t d_tuple_off_cap;
    obm_tuple *d_out; uint64_t d_out_cap;
    uint32_t *d_status; unsigned long long *d_counts;
    /* obm_lex_batch pipelines large host batches in chunks over three slots: H2D of chunk k+1, scan of
     * chunk k and D2H of chunk k-1 overlap (each slot has its own stream, staging and scratch) */
    struct Slot {
        cudaStream_t st; cudaEvent_t ev_scan; cudaEvent_t ev_k0, ev_k1; /* around the chunk's scan kernels (timing); obm_parse_batch
                                                                            records them again around parse + gather */
        uint8_t *d_bytes; uint64_t d_bytes_cap;
        uint64_t *d_doc_off; uint64_t d_doc_off_cap;
        uint64_t *d_tuple_off; uint64_t d_tuple_off_cap;
        obm_tuple *d_out; uint64_t d_out_cap;
        void *scratch; uint64_t scratch_bytes;
        uint32_t *d_status; unsigned long long *d_counts;
        /* obm_parse_batch: the chunk's records, offsets, fallback tuples and {results, args} totals */
        obm_result *d_res; uint64_t d_res_cap;
        obm_arg *d_args; uint64_t d_args_cap;
        uint64_t *d_res_off; uint64_t d_res_off_cap;
        uint64_t *d_host_off; uint64_t d_host_off_cap;
        obm_tuple *d_host; uint64_t d_host_cap;
        uint32_t *d_host_cnt; uint64_t d_host_cnt_cap;
        uint64_t *d_host_sums; uint64_t d_host_sums_cap;
        uint64_t *d_ptot; uint64_t d_ptot_cap;
        uint64_t *h_doc_off; uint64_t h_doc_off_cap; /* pinned: rebased offsets of the chunk */
        uint64_t *h_info;                             /* pinned: [0] total, [1..2] status words, [3..4] counts,
                                                         obm_parse_batch: [5..7] results, args, fallback tuples */
        uint32_t d0, d1; uint64_t b0; bool busy;
    } slots[3];
    bool slots_ready;
    uint64_t chunk_bytes; /* host batches of at least twice this size are pipelined in chunks */
    int mode; /* 0 = two-stage pipeline, 1 = exact path only, 2 = fused tile kernel */
    uint32_t launches; /* kernels launched by the last obm_lex_batch_device call */
};

static char g_static_err[256] = "no error";

static void set_err(obm_handle *h, const char *fmt, ...) {
    char *dst = h ? h->err : g_static_err; size_t cap = h ? sizeof h->err : sizeof g_static_err;
    va_list ap; va_start(ap, fmt); vsnprintf(dst, cap, fmt, ap); va_end(ap);
}

#define OBM_CUDA(h, call)                                                                              \
    do { cudaError_t e_ = (call);                                                                      \
         if (e_ != cudaSuccess) { set_err((h), "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
                                  return OBM_E_CUDA; } } while (0)

extern "C" int obm_abi_version(void) { return OBM_ABI_VERSION; }

extern "C" const char *obm_last_error(const obm_handle *h) { return h ? h->err : g_static_err; }

extern "C" int obm_create(int device_ordinal, obm_handle **out) {
    if (!out) return OBM_E_ARG;
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0) {
        set_err(nullptr, "no usable CUDA device (%s); libobmarkers has no CPU fallback", e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
        return OBM_E_NO_DEVICE;
    }
    if (device_ordinal < 0 || device_ordinal >= ndev) { set_err(nullptr, "device ordinal %d out of range (0..%d)", device_ordinal, ndev - 1); return OBM_E_ARG; }
    obm_handle *h = new (std::nothrow) obm_handle();
    if (!h) return OBM_E_NOMEM;
    memset(h, 0, sizeof *h);
    h->device = device_ordinal;
    snprintf(h->err, sizeof h->err, "no error");
    if (cudaSetDevice(device_ordinal) != cudaSuccess || cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess) {
        set_err(nullptr, "cannot initialise CUDA device %d: %s", device_ordinal, cudaGetErrorString(cudaGetLastError()));
        delete h; return OBM_E_CUDA;
    }
    for (int i = 0; i < 4; i++) cudaEventCreate(&h->ev[i]);
    cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking);
    cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming); cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming);
    if (cudaMalloc(&h->d_status, 4 * sizeof(uint32_t)) != cudaSuccess || cudaMalloc(&h->d_counts, 2 * sizeof(unsigned long long)) != cudaSuccess) {
        set_err(nullptr, "cudaMalloc failed: %s", cudaGetErrorString(cudaGetLastError()));
        delete h; return OBM_E_CUDA;
    }
    { const char *e = getenv("OBM_CHUNK_MB"); h->chunk_bytes = (uint64_t)(e && atoi(e) > 0 ? atoi(e) : 64) << 20; }
    const char *m = getenv("OBM_FORCE_EXACT");
    h->mode = (m && m[0] == '1') ? 1 : 0;
    *out = h;
    return OBM_OK;
}

extern "C" void obm_destroy(obm_handle *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    cudaFree(h->scratch); cudaFree(h->d_bytes); cudaFree(h->d_doc_off); cudaFree(h->d_tuple_off); cudaFree(h->d_out);
    cudaFree(h->d_status); cudaFree(h->d_counts);
    if (h->slots_ready) for (auto &sl : h->slots) {
        cudaStreamSynchronize(sl.st);
        cudaFree(sl.d_bytes); cudaFree(sl.d_doc_off); cudaFree(sl.d_tuple_off); cudaFree(sl.d_out); cudaFree(sl.scratch);
        cudaFree(sl.d_status); cudaFree(sl.d_counts); cudaFreeHost(sl.h_doc_off); cudaFreeHost(sl.h_info);
        cudaFree(sl.d_res); cudaFree(sl.d_args); cudaFree(sl.d_res_off); cudaFree(sl.d_host_off); cudaFree(sl.d_host);
        cudaFree(sl.d_host_cnt); cudaFree(sl.d_host_sums); cudaFree(sl.d_ptot);
        cudaEventDestroy(sl.ev_scan); cudaEventDestroy(sl.ev_k0); cudaEventDestroy(sl.ev_k1); cudaStreamDestroy(sl.st);
    }
    for (int i = 0; i < 4; i++) cudaEventDestroy(h->ev[i]);
    cudaEventDestroy(h->ev_fork); cudaEventDestroy(h->ev_join); cudaStreamDestroy(h->side);
    cudaStreamDestroy(h->stream);
    delete h;
}

/* Number of this library's kernels the last obm_lex_batch_device / obm_lex_batch call launched. */
extern "C" uint32_t obm_launches_last_call(const obm_handle *h) { return h ? h->launches : 0; }

#ifdef OBMW_PHASE_CLOCKS
/* the phase-clock build only: k_warp_scan's cycles per bucket (obmw::PC_*, summed over warps) and, at [PC_N], the units,
 * accumulated over every launch on the current device since the last reset; reset != 0 zeroes them after the read */
extern "C" int obm_phase_cycles(unsigned long long *out, int reset) {
    if (cudaDeviceSynchronize() != cudaSuccess) return OBM_E_CUDA;
    if (out && cudaMemcpyFromSymbol(out, obmw::g_phase_cycles, sizeof(obmw::g_phase_cycles)) != cudaSuccess) return OBM_E_CUDA;
    if (reset) {
        const unsigned long long z[obmw::PC_N + 1] = {};
        if (cudaMemcpyToSymbol(obmw::g_phase_cycles, z, sizeof(z)) != cudaSuccess) return OBM_E_CUDA;
    }
    return OBM_OK;
}
extern "C" int obm_phase_buckets(void) { return (int)obmw::PC_N; }
#endif

/* Chunk size of the overlapped host path (obm_lex_batch pipelines batches of >= 2 chunks). Returns the old value. */
extern "C" uint64_t obm_set_chunk_bytes(obm_handle *h, uint64_t bytes) { uint64_t old = h->chunk_bytes; if (bytes >= 4096) h->chunk_bytes = bytes; return old; }

/* Selects the scanning strategy: 0 = auto (default), 1 = exact path only. Returns the previous mode. */
extern "C" int obm_set_mode(obm_handle *h, int mode) { int old = h->mode; h->mode = mode; return old; }

template <class T>
static int ensure(obm_handle *h, T **p, uint64_t *cap, uint64_t need) {
    if (*cap >= need && *p) return OBM_OK;
    if (*p) { cudaFree(*p); *p = nullptr; *cap = 0; }
    uint64_t want = need + need / 8 + 64;
    OBM_CUDA(h, cudaMalloc((void **)p, want * sizeof(T)));
    *cap = want;
    return OBM_OK;
}

/* Fast path: index kernel -> exact count of large documents -> tile kernel -> exact fill of large documents. */
static int obm_fast_launch(obm_handle *h, void *large_ws, const uint8_t *d_bytes, const uint64_t *d_doc_off, uint32_t ndocs, uint64_t total_bytes,
                           obm_tuple *d_out, uint64_t out_cap, uint64_t *toff, uint32_t *status, unsigned long long *totals,
                           uint32_t *counts, void *ws, cudaStream_t st) {
    static bool attr_set = false;
    const size_t smem = sizeof(obmf::CtaShared);
    if (!attr_set) {
        OBM_CUDA(h, cudaFuncSetAttribute(obmf::k_tile_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_set = true;
    }
    const uint64_t nt64 = obm_fast_ntiles(total_bytes);
    if (nt64 > 0xFFFFFFF0ull) { set_err(h, "batch too large for the tile index"); return OBM_E_ARG; }
    const uint32_t ntiles = (uint32_t)nt64;
    auto up = [](uint64_t v) { return (v + 255) / 256 * 256; };
    uint8_t *w = (uint8_t *)ws;
    uint32_t *tile_first = (uint32_t *)w; w += up(((uint64_t)ntiles + 2) * 4);
    uint64_t *tile_state = (uint64_t *)w; w += up(((uint64_t)ntiles + 1) * 8);
    const uint64_t max_large = obm_fast_max_large(total_bytes);
    uint32_t *large_list = (uint32_t *)w; w += up((max_large + 1) * 4);
    uint32_t *ctl = (uint32_t *)w; /* [0] ticket, [1] n_large */
    OBM_CUDA(h, cudaMemsetAsync(tile_state, 0, ((uint64_t)ntiles + 1) * 8, st));
    OBM_CUDA(h, cudaMemsetAsync(ctl, 0, 16, st));
    obmf::k_tile_index<<<(ndocs + 1 + 255) / 256, 256, 0, st>>>(d_doc_off, ndocs, ntiles, tile_first, large_list, ctl + 1);
    int dev_sms = 0, per_sm = 0;
    OBM_CUDA(h, cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, h->device));
    const LargeWs LW = large_carve(large_ws, total_bytes, large_list, ctl + 1);
    large_count_launch(st, dev_sms, d_bytes, d_doc_off, LW, counts, totals, status);
    obmf::TileArgs A;
    A.bytes = d_bytes; A.doc_off = d_doc_off; A.ndocs = ndocs; A.total_bytes = total_bytes;
    A.tile_first = tile_first; A.ntiles = ntiles; A.counts = counts;
    A.out = d_out; A.out_cap = d_out ? out_cap : 0; A.tuple_off = toff;
    A.tile_state = tile_state; A.ticket = ctl; A.status = status; A.totals = totals;
    {
        static int msplit = -1;
        if (msplit < 0) { const char *e = getenv("OBM_MSPLIT"); msplit = e ? atoi(e) : 8; if (msplit < 1) msplit = 1; if (msplit > (int)(obmt::NT / 32)) msplit = obmt::NT / 32; }
        A.msplit = (uint32_t)msplit;
    }
    OBM_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, obmf::k_tile_scan, (int)obmt::NT, smem));
    if (per_sm < 1) per_sm = 1;
    uint32_t grid = (uint32_t)dev_sms * (uint32_t)per_sm; /* persistent CTAs: a multiple of the SM count */
    if (grid > ntiles) grid = ntiles;
    obmf::k_tile_scan<<<grid, obmt::NT, smem, st>>>(A);
    if (d_out && out_cap) large_fill_launch(st, dev_sms, d_bytes, d_doc_off, LW, toff, d_out, out_cap);
    h->launches = 2 + LARGE_COUNT_LAUNCHES + ((d_out && out_cap) ? 1 : 0);
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

static uint64_t align_up(uint64_t v, uint64_t a);
static uint32_t scan_tiles(uint32_t ndocs);

/* scratch layout: counts u32[ndocs] | tile_sums u64[ntiles] | fast-path workspace | pipeline workspace */
static uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }
static uint32_t scan_tiles(uint32_t ndocs) { return (ndocs + SCAN_TILE - 1) / SCAN_TILE; }


/* ---- two-stage pipeline (mode 0) --------------------------------------------------------------------- */
/* Structural bound, not an estimate: a unit holds at most QMAX owning lines (more -> its documents take the exact
 * lexer and contribute no line items) and an owning line is at least 2 bytes, plus one EOF item per document and
 * one item per large document.  ~0.53 B of scratch per input byte for 16 KiB tiles. */
static uint64_t pipe_items_cap(uint32_t ndocs, uint64_t total_bytes) {
    const uint64_t by_units = (obm_fast_ntiles(total_bytes) + ndocs / obmt::DMAX + 2) * (uint64_t)obmt::QMAX, by_bytes = total_bytes / 2 + 1;
    return (by_units < by_bytes ? by_units : by_bytes) + 2ull * ndocs + obm_fast_ntiles(total_bytes) + 1024;
}
static uint64_t pipe_units_max(uint32_t ndocs, uint64_t total_bytes) { return obm_fast_ntiles(total_bytes) + ndocs / obmt::DMAX + 2; }
static uint64_t pipe_scratch_bytes(uint32_t ndocs, uint64_t total_bytes) {
    const uint64_t nt = obm_fast_ntiles(total_bytes), um = pipe_units_max(ndocs, total_bytes);
    return align_up(pipe_items_cap(ndocs, total_bytes) * 8, 256) + align_up(nt * 4 + 4, 256) + align_up((nt + 1) * 8, 256) +
           align_up(((uint64_t)scan_tiles((uint32_t)nt) + 1) * 8, 256) + align_up((nt + 1) * sizeof(obmp::TileRec), 256) + align_up((um + 1) * 16, 256) +
           align_up((uint64_t)ndocs * 4 + 4, 256) + align_up((um + 1) * 8, 256) + align_up((um / 32 + 2) * 8, 256) + 256;
}

/* index -> exact count of large documents -> units per tile (+ scan) -> k1_scan -> k2_units -> exact fill of
 * large documents. */
static int obm_pipe_launch(obm_handle *h, const uint8_t *d_bytes, const uint64_t *d_doc_off, uint32_t ndocs, uint64_t total_bytes,
                            obm_tuple *d_out, uint64_t out_cap, uint64_t *toff, uint32_t *status, unsigned long long *totals,
                            uint32_t *counts, void *fast_ws, void *pipe_ws, void *large_ws, cudaStream_t st) {
    static bool attr_set = false;
    const size_t smem1 = sizeof(obmq::K1Shared);
    if (!attr_set) {
        OBM_CUDA(h, cudaFuncSetAttribute(obmq::k1_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
        attr_set = true;
    }
    const uint64_t nt64 = obm_fast_ntiles(total_bytes);
    if (nt64 > 0xFFFFFFF0ull || pipe_units_max(ndocs, total_bytes) > 0xFFFFFFF0ull) { set_err(h, "batch too large for the tile index"); return OBM_E_ARG; }
    const uint32_t ntiles = (uint32_t)nt64;
    auto up = [](uint64_t v) { return (v + 255) / 256 * 256; };
    uint8_t *w = (uint8_t *)fast_ws;
    uint32_t *tile_first = (uint32_t *)w; w += up(((uint64_t)ntiles + 2) * 4);
    w += up(((uint64_t)ntiles + 1) * 8); /* tile_state of the fused kernel: unused here */
    const uint64_t max_large = obm_fast_max_large(total_bytes);
    uint32_t *large_list = (uint32_t *)w; w += up((max_large + 1) * 4);
    uint32_t *lctl = (uint32_t *)w; /* [1] n_large */
    const uint64_t ic = pipe_items_cap(ndocs, total_bytes), um = pipe_units_max(ndocs, total_bytes);
    const uint32_t nt_u = scan_tiles(ntiles);
    uint8_t *q = (uint8_t *)pipe_ws;
    obmq::PipeArgs A;
    A.bytes = d_bytes; A.doc_off = d_doc_off; A.ndocs = ndocs; A.total_bytes = total_bytes; A.tile_first = tile_first; A.ntiles = ntiles;
    A.items = (obmp::item_t *)q; q += up(ic * 8); A.items_cap = ic;
    uint32_t *nsub = (uint32_t *)q; q += up((uint64_t)ntiles * 4 + 4);
    uint64_t *ubase = (uint64_t *)q; q += up(((uint64_t)ntiles + 1) * 8); A.ubase = ubase;
    uint64_t *usums = (uint64_t *)q; q += up(((uint64_t)nt_u + 1) * 8);
    obmp::TileRec *trec = (obmp::TileRec *)q; q += up(((uint64_t)ntiles + 1) * sizeof(obmp::TileRec)); A.trec = trec;
    A.units = (obmp::Unit *)q; q += up((um + 1) * 16);
    A.doc_flag = (uint32_t *)q; q += up((uint64_t)ndocs * 4 + 4);
    A.st_tuples = (uint64_t *)q; q += up((um + 1) * 8);
    A.st_blocks = (uint64_t *)q; q += up((um / 32 + 2) * 8);
    A.ctl = (uint32_t *)q;
    A.counts = counts; A.out = d_out; A.out_cap = d_out ? out_cap : 0; A.tuple_off = toff;
    A.status = status; A.totals = totals;
    OBM_CUDA(h, cudaMemsetAsync(A.st_tuples, 0, up((um + 1) * 8) + up((um / 32 + 2) * 8) + 64, st)); /* look-back chains + control words */
    OBM_CUDA(h, cudaMemsetAsync(lctl, 0, 16, st));
    obmf::k_tile_index<<<(ndocs + 1 + 255) / 256, 256, 0, st>>>(d_doc_off, ndocs, ntiles, tile_first, large_list, lctl + 1);
    int dev_sms = 0, per_sm1 = 0, per_sm2 = 0;
    OBM_CUDA(h, cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, h->device));
    const LargeWs LW = large_carve(large_ws, total_bytes, large_list, lctl + 1);
    /* the eight small kernels that plan and count the large documents depend only on k_tile_index and are needed
     * by k2_units: they run on a side stream under k1_scan instead of in front of it */
    OBM_CUDA(h, cudaEventRecord(h->ev_fork, st));
    OBM_CUDA(h, cudaStreamWaitEvent(h->side, h->ev_fork, 0));
    large_count_launch(h->side, dev_sms, d_bytes, d_doc_off, LW, counts, totals, status);
    OBM_CUDA(h, cudaEventRecord(h->ev_join, h->side));
    obmq::k_tile_units<<<(ntiles + 255) / 256, 256, 0, st>>>(d_doc_off, tile_first, ntiles, nsub, trec);
    k_scan_tiles<<<nt_u, SCAN_THREADS, 0, st>>>(nsub, ntiles, ubase, usums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(usums, nt_u, ubase + ntiles);
    k_scan_add<<<nt_u, SCAN_THREADS, 0, st>>>(ubase, ntiles, usums, ~0ull, nullptr);
    OBM_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm1, obmq::k1_scan, (int)obmt::NT, smem1));
    OBM_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm2, obmq::k2_units<false>, (int)(obmp::W_WARPS * 32), 0));
    if (per_sm1 < 1) per_sm1 = 1;
    if (per_sm2 < 1) per_sm2 = 1;
    uint32_t g1 = (uint32_t)dev_sms * (uint32_t)per_sm1; /* persistent CTAs: multiples of the SM count */
    if (g1 > ntiles) g1 = ntiles;
    uint32_t g2 = (uint32_t)dev_sms * (uint32_t)per_sm2;
    const uint64_t g2max = (um + obmp::W_WARPS - 1) / obmp::W_WARPS;
    if (g2 > g2max) g2 = (uint32_t)g2max;
    obmq::k1_scan<<<g1, obmt::NT, smem1, st>>>(A);
    OBM_CUDA(h, cudaStreamWaitEvent(st, h->ev_join, 0));
    obmq::k2_units<false><<<g2, obmp::W_WARPS * 32, 0, st>>>(A); /* batches without non-ASCII text */
    obmq::k2_units<true><<<g2, obmp::W_WARPS * 32, 0, st>>>(A);  /* batches with valid UTF-8 beyond ASCII: per-line Unicode lexing */
    uint32_t launches = 8 + LARGE_COUNT_LAUNCHES;
    if (d_out && out_cap) {
        large_fill_launch(st, dev_sms, d_bytes, d_doc_off, LW, toff, d_out, out_cap);
        launches += 1;
    }
    /* work-record overflow -> status[3]: the caller must redo the scan with the exact kernels (mode 1) */
    OBM_CUDA(h, cudaMemcpyAsync(status + ST_RESERVED, A.ctl + obmq::CT_OVF, sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
    h->launches = launches;
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

/* ---- fused warp kernel (mode 0) ----------------------------------------------------------------------- */
static uint64_t warp_ntiles(uint64_t total_bytes) { return total_bytes / obmw::TILE + 1; }
static uint64_t warp_units_max(uint32_t ndocs, uint64_t total_bytes) { return 2 * warp_ntiles(total_bytes) + ndocs / obmw::DMAX + 2; }
static uint64_t warp_scratch_bytes(uint32_t ndocs, uint64_t total_bytes) {
    const uint64_t nt = warp_ntiles(total_bytes), um = warp_units_max(ndocs, total_bytes);
    return align_up((nt + 2) * 4, 256) + align_up((obm_fast_max_large(total_bytes) + 1) * 4, 256) + align_up(nt * 4 + 4, 256) + align_up((nt + 1) * 8, 256) +
           align_up(((uint64_t)scan_tiles((uint32_t)nt) + 1) * 8, 256) + align_up((nt + 1) * sizeof(obmw::WRec), 256) + align_up((um + 1) * 8, 256) +
           align_up(2 * (um / 32 + 2) * 8, 256) + align_up((um + 1) * 4, 256) + 512;
}
/* tile index -> (large documents planned and counted on a side stream) units per tile + scan -> k_warp_scan -> fill of
 * the large documents */
static int obm_warp_launch(obm_handle *h, const uint8_t *d_bytes, const uint64_t *d_doc_off, uint32_t ndocs, uint64_t total_bytes,
                           obm_tuple *d_out, uint64_t out_cap, uint64_t *toff, uint32_t *status, unsigned long long *totals,
                           uint32_t *counts, void *warp_ws, void *large_ws, cudaStream_t st) {
    static_assert(sizeof(obmw::WarpSmem) * obmw::WPC <= 232448, "the warps of the CTA share the 227 KB of one SM");
    const size_t smem = sizeof(obmw::WarpSmem) * obmw::WPC;
    OBM_CUDA(h, cudaFuncSetAttribute(obmw::k_warp_scan, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); /* per device: set on every call (cheap) */
    const uint64_t nt64 = warp_ntiles(total_bytes), um = warp_units_max(ndocs, total_bytes);
    if (nt64 > 0xFFFFFFF0ull || um > 0xFFFFFFF0ull) { set_err(h, "batch too large for the tile index"); return OBM_E_ARG; }
    const uint32_t ntiles = (uint32_t)nt64, nt_u = scan_tiles(ntiles);
    auto up = [](uint64_t v) { return (v + 255) / 256 * 256; };
    uint8_t *q = (uint8_t *)warp_ws;
    uint32_t *tile_first = (uint32_t *)q; q += up(((uint64_t)ntiles + 2) * 4);
    uint32_t *large_list = (uint32_t *)q; q += up((obm_fast_max_large(total_bytes) + 1) * 4);
    uint32_t *nun = (uint32_t *)q; q += up((uint64_t)ntiles * 4 + 4);
    uint64_t *ubase = (uint64_t *)q; q += up(((uint64_t)ntiles + 1) * 8);
    uint64_t *usums = (uint64_t *)q; q += up(((uint64_t)nt_u + 1) * 8);
    obmw::WRec *wrec = (obmw::WRec *)q; q += up(((uint64_t)ntiles + 1) * sizeof(obmw::WRec));
    uint32_t *unit_tile = (uint32_t *)q; q += up((um + 1) * 4);
    obmw::WArgs A;
    A.unit_tile = unit_tile;
    A.bytes = d_bytes; A.doc_off = d_doc_off; A.ndocs = ndocs; A.total_bytes = total_bytes; A.tile_first = tile_first; A.ntiles = ntiles;
    A.wrec = wrec; A.ubase = ubase;
    A.st_tuples = (uint64_t *)q; q += up((um + 1) * 8);
    A.st_blocks = (uint64_t *)q; q += up(2 * (um / 32 + 2) * 8); A.units_max = um;
    A.ctl = (uint32_t *)q; /* [0] ticket, [1] n_large */
    A.counts = counts; A.out = d_out; A.out_cap = d_out ? out_cap : 0; A.tuple_off = toff; A.status = status; A.totals = totals;
    OBM_CUDA(h, cudaMemsetAsync(A.st_tuples, 0, up((um + 1) * 8) + up(2 * (um / 32 + 2) * 8) + 64, st)); /* chain arrays + control words */
    obmw::k_wtile_index<<<(ndocs + 1 + 255) / 256, 256, 0, st>>>(d_doc_off, ndocs, ntiles, tile_first, large_list, A.ctl + 1);
    int dev_sms = 0, per_sm = 0;
    OBM_CUDA(h, cudaDeviceGetAttribute(&dev_sms, cudaDevAttrMultiProcessorCount, h->device));
    const LargeWs LW = large_carve(large_ws, total_bytes, large_list, A.ctl + 1);
    OBM_CUDA(h, cudaEventRecord(h->ev_fork, st));
    OBM_CUDA(h, cudaStreamWaitEvent(h->side, h->ev_fork, 0));
    large_count_launch(h->side, dev_sms, d_bytes, d_doc_off, LW, counts, totals, status);
    OBM_CUDA(h, cudaEventRecord(h->ev_join, h->side));
    obmw::k_wunits<<<(ntiles + 255) / 256, 256, 0, st>>>(d_doc_off, tile_first, ntiles, nun, wrec);
    k_scan_tiles<<<nt_u, SCAN_THREADS, 0, st>>>(nun, ntiles, ubase, usums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(usums, nt_u, ubase + ntiles);
    k_scan_add<<<nt_u, SCAN_THREADS, 0, st>>>(ubase, ntiles, usums, ~0ull, nullptr);
    obmw::k_wunit_tiles<<<(ntiles + 255) / 256, 256, 0, st>>>(nun, ubase, ntiles, um, unit_tile);
    OBM_CUDA(h, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, obmw::k_warp_scan, (int)(obmw::WPC * 32), smem));
    if (per_sm < 1) per_sm = 1;
    uint32_t grid = (uint32_t)dev_sms * (uint32_t)per_sm; /* persistent warps: a multiple of the SM count */
    const uint32_t gmax = (uint32_t)((um < 0xFFFFFFF0ull ? um : 0xFFFFFFF0ull) + obmw::WPC - 1) / obmw::WPC;
    if (grid > gmax) grid = gmax;
    OBM_CUDA(h, cudaStreamWaitEvent(st, h->ev_join, 0));
    obmw::k_warp_scan<<<grid, obmw::WPC * 32, smem, st>>>(A);
    uint32_t launches = 7 + LARGE_COUNT_LAUNCHES;
    if (d_out && out_cap) { large_fill_launch(st, dev_sms, d_bytes, d_doc_off, LW, toff, d_out, out_cap); launches += 1; }
    h->launches = launches;
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

extern "C" uint64_t obm_scratch_bytes(uint32_t ndocs, uint64_t total_bytes) {
    uint64_t b = align_up((uint64_t)ndocs * 4 + 4, 256);
    b += align_up((uint64_t)scan_tiles(ndocs) * 8 + 8, 256);
    b += align_up(obm_fast_scratch_bytes(ndocs, total_bytes), 256);
    b += pipe_scratch_bytes(ndocs, total_bytes);
    b += large_scratch_bytes(total_bytes);
    b += warp_scratch_bytes(ndocs, total_bytes);
    return b;
}

static int lex_device_impl(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                           uint64_t total_bytes, void *d_out, uint64_t out_cap, void *d_doc_tuple_off,
                           void *d_status, void *d_counts, cudaStream_t st, void **scratch_p = nullptr, uint64_t *scratch_bytes_p = nullptr) {
    if (!h) return OBM_E_ARG;
    if (!d_doc_off || !d_doc_tuple_off || (ndocs && total_bytes && !d_bytes)) { set_err(h, "null device pointer"); return OBM_E_ARG; }
    OBM_CUDA(h, cudaSetDevice(h->device));
    if (!scratch_p) { scratch_p = &h->scratch; scratch_bytes_p = &h->scratch_bytes; }
    uint64_t need = obm_scratch_bytes(ndocs, total_bytes);
    if (*scratch_bytes_p < need) {
        if (*scratch_p) { OBM_CUDA(h, cudaStreamSynchronize(st)); cudaFree(*scratch_p); *scratch_p = nullptr; *scratch_bytes_p = 0; }
        OBM_CUDA(h, cudaMalloc(scratch_p, need));
        *scratch_bytes_p = need;
    }
    uint8_t *sc = (uint8_t *)*scratch_p;
    uint32_t *counts = (uint32_t *)sc; sc += align_up((uint64_t)ndocs * 4 + 4, 256);
    uint64_t *tile_sums = (uint64_t *)sc; sc += align_up((uint64_t)scan_tiles(ndocs) * 8 + 8, 256);
    void *fast_ws = sc; sc += align_up(obm_fast_scratch_bytes(ndocs, total_bytes), 256);
    void *pipe_ws = sc; sc += pipe_scratch_bytes(ndocs, total_bytes);
    void *large_ws = sc; sc += large_scratch_bytes(total_bytes);
    void *warp_ws = sc;
    uint32_t *status = (uint32_t *)(d_status ? d_status : (void *)h->d_status);
    unsigned long long *totals = (unsigned long long *)(d_counts ? d_counts : (void *)h->d_counts);
    uint64_t *toff = (uint64_t *)d_doc_tuple_off;
    OBM_CUDA(h, cudaMemsetAsync(status, 0, 4 * sizeof(uint32_t), st));
    OBM_CUDA(h, cudaMemsetAsync(totals, 0, 2 * sizeof(unsigned long long), st));
    if (ndocs == 0) { OBM_CUDA(h, cudaMemsetAsync(toff, 0, sizeof(uint64_t), st)); return OBM_OK; }

    if (h->mode == 0)
        return obm_warp_launch(h, (const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, total_bytes, (obm_tuple *)d_out, out_cap, toff, status,
                               totals, counts, warp_ws, large_ws, st);
    if (h->mode == 3)
        return obm_pipe_launch(h, (const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, total_bytes,
                                (obm_tuple *)d_out, out_cap, toff, status, totals, counts, fast_ws, pipe_ws, large_ws, st);
    if (h->mode == 2)
        return obm_fast_launch(h, large_ws, (const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, total_bytes,
                               (obm_tuple *)d_out, out_cap, toff, status, totals, counts, fast_ws, st);
    uint32_t nb = (ndocs + 127) / 128;
    h->launches = 4 + ((d_out && out_cap) ? 1 : 0);
    k_exact_count<<<nb, 128, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, nullptr, ndocs, nullptr, counts, totals, status);
    uint32_t nt = scan_tiles(ndocs);
    k_scan_tiles<<<nt, SCAN_THREADS, 0, st>>>(counts, ndocs, toff, tile_sums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(tile_sums, nt, toff + ndocs);
    k_scan_add<<<nt, SCAN_THREADS, 0, st>>>(toff, ndocs, tile_sums, out_cap, status);
    if (d_out && out_cap)
        k_exact_fill<<<nb, 128, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, nullptr, ndocs, nullptr, toff, (obm_tuple *)d_out, out_cap);
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

/* `stream` is used exactly as given: NULL is CUDA's (legacy) default stream, like any CUDA API. */
extern "C" int obm_lex_batch_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                                    uint64_t total_bytes, void *d_out, uint64_t out_cap, void *d_doc_tuple_off,
                                    void *d_status, void *d_counts, void *stream) {
    return lex_device_impl(h, d_bytes, d_doc_off, ndocs, total_bytes, d_out, out_cap, d_doc_tuple_off, d_status, d_counts,
                           (cudaStream_t)stream);
}


/* ---- chunked, overlapped host path ------------------------------------------------------------------- */
static int slots_init(obm_handle *h) {
    if (h->slots_ready) return OBM_OK;
    for (auto &sl : h->slots) {
        memset(&sl, 0, sizeof sl);
        OBM_CUDA(h, cudaStreamCreateWithFlags(&sl.st, cudaStreamNonBlocking));
        OBM_CUDA(h, cudaEventCreateWithFlags(&sl.ev_scan, cudaEventDisableTiming));
        OBM_CUDA(h, cudaEventCreate(&sl.ev_k0)); OBM_CUDA(h, cudaEventCreate(&sl.ev_k1));
        OBM_CUDA(h, cudaMalloc(&sl.d_status, 4 * sizeof(uint32_t)));
        OBM_CUDA(h, cudaMalloc(&sl.d_counts, 2 * sizeof(unsigned long long)));
        OBM_CUDA(h, cudaHostAlloc((void **)&sl.h_info, 8 * sizeof(uint64_t), cudaHostAllocDefault));
    }
    h->slots_ready = true;
    return OBM_OK;
}

/* enqueue the scan of the slot's staged chunk (nb bytes) + the D2H of its info words */
static int chunk_scan(obm_handle *h, obm_handle::Slot &sl, uint64_t nb, bool want_out) {
    const uint32_t nd = sl.d1 - sl.d0;
    OBM_CUDA(h, cudaEventRecord(sl.ev_k0, sl.st));
    int rc = lex_device_impl(h, sl.d_bytes, sl.d_doc_off, nd, nb, want_out ? sl.d_out : nullptr, want_out ? sl.d_out_cap : 0, sl.d_tuple_off,
                             sl.d_status, sl.d_counts, sl.st, &sl.scratch, &sl.scratch_bytes);
    if (rc != OBM_OK) return rc;
    OBM_CUDA(h, cudaEventRecord(sl.ev_k1, sl.st));
    OBM_CUDA(h, cudaMemcpyAsync(&sl.h_info[0], sl.d_tuple_off + nd, 8, cudaMemcpyDeviceToHost, sl.st));
    OBM_CUDA(h, cudaMemcpyAsync(&sl.h_info[1], sl.d_status, 16, cudaMemcpyDeviceToHost, sl.st));
    OBM_CUDA(h, cudaMemcpyAsync(&sl.h_info[3], sl.d_counts, 16, cudaMemcpyDeviceToHost, sl.st));
    OBM_CUDA(h, cudaEventRecord(sl.ev_scan, sl.st));
    return OBM_OK;
}

/* enqueue H2D + scan + info D2H of documents [d0, d1) on slot sl */
static int chunk_issue(obm_handle *h, obm_handle::Slot &sl, const uint8_t *bytes, const uint64_t *doc_off, uint32_t d0, uint32_t d1,
                       bool want_out) {
    const uint32_t nd = d1 - d0;
    const uint64_t b0 = doc_off[d0], nb = doc_off[d1] - b0;
    int rc;
    if ((rc = ensure(h, &sl.d_bytes, &sl.d_bytes_cap, nb + 64)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_doc_off, &sl.d_doc_off_cap, (uint64_t)nd + 1)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_tuple_off, &sl.d_tuple_off_cap, (uint64_t)nd + 1)) != OBM_OK) return rc;
    const uint64_t cap = want_out ? nb / 4 + 2ull * nd + 1024 : 0; /* 2 B of tuples per input byte: ~6x what manifests need */
    if (want_out && (rc = ensure(h, &sl.d_out, &sl.d_out_cap, cap)) != OBM_OK) return rc;
    if (sl.h_doc_off_cap < (uint64_t)nd + 1) {
        if (sl.h_doc_off) cudaFreeHost(sl.h_doc_off);
        sl.h_doc_off = nullptr; sl.h_doc_off_cap = 0;
        uint64_t want = (uint64_t)nd + 1 + nd / 8 + 64;
        OBM_CUDA(h, cudaHostAlloc((void **)&sl.h_doc_off, want * 8, cudaHostAllocDefault));
        sl.h_doc_off_cap = want;
    }
    for (uint32_t d = 0; d <= nd; d++) sl.h_doc_off[d] = doc_off[d0 + d] - b0;
    OBM_CUDA(h, cudaMemcpyAsync(sl.d_doc_off, sl.h_doc_off, ((uint64_t)nd + 1) * 8, cudaMemcpyHostToDevice, sl.st));
    if (nb) OBM_CUDA(h, cudaMemcpyAsync(sl.d_bytes, bytes + b0, nb, cudaMemcpyHostToDevice, sl.st));
    sl.d0 = d0; sl.d1 = d1; sl.b0 = b0; sl.busy = true;
    return chunk_scan(h, sl, nb, want_out);
}

struct ChunkTotals { uint64_t tuples, markers, lexemes, exact, fatal; bool overflow, need_exact; float ms_kernels; };

/* wait for the slot's scan, then enqueue the D2H of its tuples / offsets at their final host positions */
static int chunk_retire(obm_handle *h, obm_handle::Slot &sl, obm_tuple *out, uint64_t out_cap, uint64_t *doc_tuple_off,
                        uint64_t *chunk_base /* per document's chunk base, filled for the fix-up */, ChunkTotals &T) {
    OBM_CUDA(h, cudaEventSynchronize(sl.ev_scan));
    { float ms = 0.f; if (cudaEventElapsedTime(&ms, sl.ev_k0, sl.ev_k1) == cudaSuccess) T.ms_kernels += ms; }
    const uint32_t nd = sl.d1 - sl.d0;
    const uint64_t total = sl.h_info[0];
    const uint32_t *st = (const uint32_t *)&sl.h_info[1];
    if (st[ST_RESERVED]) T.need_exact = true;       /* work-record overflow: the caller redoes the batch with the exact kernels */
    if (st[ST_OVERFLOW] && out) T.overflow = true;  /* the slot's tuple buffer was too small for this chunk */
    const uint64_t base = T.tuples;
    *chunk_base = base;
    OBM_CUDA(h, cudaMemcpyAsync(doc_tuple_off + sl.d0, sl.d_tuple_off, (uint64_t)nd * 8, cudaMemcpyDeviceToHost, sl.st));
    if (out && !T.overflow && !T.need_exact && base + total <= out_cap && total)
        OBM_CUDA(h, cudaMemcpyAsync(out + base, sl.d_out, total * sizeof(obm_tuple), cudaMemcpyDeviceToHost, sl.st));
    T.tuples += total; T.markers += sl.h_info[3]; T.lexemes += sl.h_info[4]; T.exact += st[ST_DOCS_EXACT]; T.fatal += st[ST_DOCS_FATAL];
    sl.busy = false;
    return OBM_OK;
}

/* chunk boundaries (document aligned: a chunk ends before the first document that would take it past chunk_bytes, and
 * holds at least one document) and the per-chunk base for the final offset fix-up; malloc'd, NULL when out of memory */
struct Ck { uint32_t d0, d1; uint64_t base; };
static Ck *cut_chunks(const uint64_t *doc_off, uint32_t ndocs, uint64_t chunk_bytes, uint32_t *nck) {
    Ck *cks = nullptr; uint32_t n = 0, capck = 0;
    for (uint32_t d = 0; d < ndocs;) {
        uint32_t e = d; const uint64_t lim = doc_off[d] + chunk_bytes;
        while (e < ndocs && (doc_off[e + 1] <= lim || e == d)) e++;
        if (n == capck) {
            capck = capck ? capck * 2 : 64;
            Ck *g = (Ck *)realloc(cks, capck * sizeof(Ck));
            if (!g) { free(cks); return nullptr; }
            cks = g;
        }
        cks[n++] = Ck{d, e, 0};
        d = e;
    }
    if (!cks) cks = (Ck *)malloc(sizeof(Ck));
    *nck = n;
    return cks;
}

/* the host entry points' checks of a packed batch: ascending offsets, documents within OBM_MAX_DOC_BYTES, bytes given */
static int check_host_batch(obm_handle *h, const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs) {
    for (uint32_t d = 0; d < ndocs; d++) {
        if (doc_off[d + 1] < doc_off[d]) { set_err(h, "doc_off is not ascending at document %u", d); return OBM_E_ARG; }
        if (doc_off[d + 1] - doc_off[d] > OBM_MAX_DOC_BYTES) { set_err(h, "document %u exceeds %llu bytes", d, (unsigned long long)OBM_MAX_DOC_BYTES); return OBM_E_ARG; }
    }
    if (doc_off[ndocs] > doc_off[0] && !bytes) { set_err(h, "bytes is NULL"); return OBM_E_ARG; }
    return OBM_OK;
}

/* returns 1 when the batch was handled here, 0 to let the caller use the single-shot path, <0 on error */
static int lex_batch_chunked(obm_handle *h, const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs, obm_tuple *out, uint64_t out_cap,
                             uint64_t *out_count, uint64_t *doc_tuple_off, obm_stats *stats, int *result) {
    const uint64_t chunk_bytes = h->chunk_bytes;
    const uint64_t total = doc_off[ndocs] - doc_off[0];
    if (total < 2 * chunk_bytes || ndocs < 4) return 0;
    int rc;
    if ((rc = slots_init(h)) != OBM_OK) return rc;
    OBM_CUDA(h, cudaEventRecord(h->ev[0], h->stream));
    ChunkTotals T = {0, 0, 0, 0, 0, false, false, 0.f};
    uint32_t nck = 0;
    Ck *cks = cut_chunks(doc_off, ndocs, chunk_bytes, &nck);
    if (!cks) return OBM_E_NOMEM;
    int err = OBM_OK;
    for (uint32_t k = 0; k < nck + 2 && err == OBM_OK; k++) {
        if (k < nck) {
            obm_handle::Slot &sl = h->slots[k % 3];
            /* the slot's previous chunk (k-3) was retired two iterations ago; its D2H copies are still queued on the
             * slot's stream, in order, ahead of this chunk's H2D -- only the pinned offsets staging needs the host to wait */
            if (k >= 3) { cudaError_t e_ = cudaStreamSynchronize(sl.st); if (e_ != cudaSuccess) { set_err(h, "cudaStreamSynchronize failed: %s", cudaGetErrorString(e_)); err = OBM_E_CUDA; break; } }
            err = chunk_issue(h, sl, bytes, doc_off, cks[k].d0, cks[k].d1, out != nullptr && out_cap > 0);
            if (err != OBM_OK) break;
        }
        if (k >= 2 && k - 2 < nck) err = chunk_retire(h, h->slots[(k - 2) % 3], out, out_cap, doc_tuple_off, &cks[k - 2].base, T);
    }
    for (auto &sl : h->slots) cudaStreamSynchronize(sl.st);
    if (err != OBM_OK) { free(cks); return err; }
    if (T.need_exact || T.overflow) { free(cks); return 0; } /* rare: let the single-shot path (with its own fallbacks) redo the batch */
    for (uint32_t k = 0; k < nck; k++) { const uint64_t b = cks[k].base; if (b) for (uint32_t d = cks[k].d0; d < cks[k].d1; d++) doc_tuple_off[d] += b; }
    free(cks);
    doc_tuple_off[ndocs] = T.tuples;
    *out_count = T.tuples;
    *result = OBM_OK;
    if (T.tuples > out_cap || (!out && T.tuples > 0)) {
        set_err(h, "output capacity %llu < %llu tuples required", (unsigned long long)out_cap, (unsigned long long)T.tuples);
        *result = OBM_E_CAPACITY;
    }
    OBM_CUDA(h, cudaEventRecord(h->ev[3], h->stream));
    OBM_CUDA(h, cudaStreamSynchronize(h->stream));
    if (stats) {
        memset(stats, 0, sizeof *stats);
        stats->n_tuples = T.tuples; stats->n_markers = T.markers; stats->n_lexemes = T.lexemes;
        stats->n_docs_exact = T.exact; stats->n_docs_fatal = T.fatal; stats->bytes = total;
        cudaEventElapsedTime(&stats->ms_total, h->ev[0], h->ev[3]);
        stats->ms_kernels = T.ms_kernels; /* sum over the chunks (their scans overlap the copies of other chunks) */
    }
    return 1;
}

extern "C" int obm_lex_batch(obm_handle *h, const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs,
                             obm_tuple *out, uint64_t out_cap, uint64_t *out_count, uint64_t *doc_tuple_off,
                             obm_stats *stats) {
    if (!h) return OBM_E_ARG;
    if (!doc_off || !out_count || !doc_tuple_off) { set_err(h, "doc_off, out_count and doc_tuple_off must not be NULL"); return OBM_E_ARG; }
    int rc;
    if ((rc = check_host_batch(h, bytes, doc_off, ndocs)) != OBM_OK) return rc;
    uint64_t total = doc_off[ndocs] - doc_off[0];
    OBM_CUDA(h, cudaSetDevice(h->device));
    cudaStream_t st = h->stream;
    {
        int result = OBM_OK;
        rc = lex_batch_chunked(h, bytes, doc_off, ndocs, out, out_cap, out_count, doc_tuple_off, stats, &result);
        if (rc < 0) return rc;
        if (rc == 1) return result;
    }
    if ((rc = ensure(h, &h->d_bytes, &h->d_bytes_cap, total + 64)) != OBM_OK) return rc;
    if ((rc = ensure(h, &h->d_doc_off, &h->d_doc_off_cap, (uint64_t)ndocs + 1)) != OBM_OK) return rc;
    if ((rc = ensure(h, &h->d_tuple_off, &h->d_tuple_off_cap, (uint64_t)ndocs + 1)) != OBM_OK) return rc;
    /* device output sized for the caller's capacity, but at least a typical 0.5 tuples/byte guess so
     * that a sizing call followed by the real call does not reallocate */
    uint64_t want_out = out_cap;
    if ((rc = ensure(h, &h->d_out, &h->d_out_cap, want_out + 1)) != OBM_OK) return rc;

    OBM_CUDA(h, cudaEventRecord(h->ev[0], st));
    /* rebase offsets so that the device batch starts at 0 */
    const uint64_t base = doc_off[0];
    if (base == 0) {
        OBM_CUDA(h, cudaMemcpyAsync(h->d_doc_off, doc_off, ((uint64_t)ndocs + 1) * 8, cudaMemcpyHostToDevice, st));
    } else {
        uint64_t *tmp = (uint64_t *)malloc(((uint64_t)ndocs + 1) * 8);
        if (!tmp) return OBM_E_NOMEM;
        for (uint32_t d = 0; d <= ndocs; d++) tmp[d] = doc_off[d] - base;
        cudaError_t e = cudaMemcpyAsync(h->d_doc_off, tmp, ((uint64_t)ndocs + 1) * 8, cudaMemcpyHostToDevice, st);
        cudaStreamSynchronize(st);
        free(tmp);
        OBM_CUDA(h, e);
    }
    if (total) OBM_CUDA(h, cudaMemcpyAsync(h->d_bytes, bytes + base, total, cudaMemcpyHostToDevice, st));
    OBM_CUDA(h, cudaEventRecord(h->ev[1], st));
    rc = lex_device_impl(h, h->d_bytes, h->d_doc_off, ndocs, total, (out && out_cap) ? h->d_out : nullptr, out_cap,
                         h->d_tuple_off, nullptr, nullptr, st);
    if (rc != OBM_OK) return rc;
    OBM_CUDA(h, cudaEventRecord(h->ev[2], st));
    OBM_CUDA(h, cudaMemcpyAsync(doc_tuple_off, h->d_tuple_off, ((uint64_t)ndocs + 1) * 8, cudaMemcpyDeviceToHost, st));
    uint32_t hstatus[4]; unsigned long long hcounts[2];
    OBM_CUDA(h, cudaMemcpyAsync(hstatus, h->d_status, sizeof hstatus, cudaMemcpyDeviceToHost, st));
    OBM_CUDA(h, cudaMemcpyAsync(hcounts, h->d_counts, sizeof hcounts, cudaMemcpyDeviceToHost, st));
    OBM_CUDA(h, cudaStreamSynchronize(st));
    if (hstatus[ST_RESERVED] && h->mode != 1) {
        /* the pipeline's work-record buffers overflowed (input far denser in markers than manifests are):
         * redo this batch with the exact kernels, which have no such limit */
        const int saved = h->mode;
        h->mode = 1;
        rc = lex_device_impl(h, h->d_bytes, h->d_doc_off, ndocs, total, (out && out_cap) ? h->d_out : nullptr, out_cap,
                             h->d_tuple_off, nullptr, nullptr, st);
        h->mode = saved;
        if (rc != OBM_OK) return rc;
        OBM_CUDA(h, cudaEventRecord(h->ev[2], st));
        OBM_CUDA(h, cudaMemcpyAsync(doc_tuple_off, h->d_tuple_off, ((uint64_t)ndocs + 1) * 8, cudaMemcpyDeviceToHost, st));
        OBM_CUDA(h, cudaMemcpyAsync(hstatus, h->d_status, sizeof hstatus, cudaMemcpyDeviceToHost, st));
        OBM_CUDA(h, cudaMemcpyAsync(hcounts, h->d_counts, sizeof hcounts, cudaMemcpyDeviceToHost, st));
        OBM_CUDA(h, cudaStreamSynchronize(st));
    }
    uint64_t ntup = doc_tuple_off[ndocs];
    *out_count = ntup;
    int result = OBM_OK;
    if (ntup > out_cap || (!out && ntup > 0)) {
        set_err(h, "output capacity %llu < %llu tuples required", (unsigned long long)out_cap, (unsigned long long)ntup);
        result = OBM_E_CAPACITY;
    } else if (ntup) {
        OBM_CUDA(h, cudaMemcpyAsync(out, h->d_out, ntup * sizeof(obm_tuple), cudaMemcpyDeviceToHost, st));
    }
    OBM_CUDA(h, cudaEventRecord(h->ev[3], st));
    OBM_CUDA(h, cudaStreamSynchronize(st));
    if (stats) {
        memset(stats, 0, sizeof *stats);
        stats->n_tuples = ntup; stats->n_markers = hcounts[0]; stats->n_lexemes = hcounts[1];
        stats->n_docs_exact = hstatus[ST_DOCS_EXACT]; stats->n_docs_fatal = hstatus[ST_DOCS_FATAL];
        stats->bytes = total;
        cudaEventElapsedTime(&stats->ms_kernels, h->ev[1], h->ev[2]);
        cudaEventElapsedTime(&stats->ms_total, h->ev[0], h->ev[3]);
    }
    return result;
}

extern "C" int obm_generate_corpus_device(obm_handle *h, void *d_bytes, void *d_doc_off, uint32_t ndocs,
                                          uint32_t doc_bytes, uint64_t first_doc, int flavour, void *stream_v) {
    if (!h || !d_bytes) return OBM_E_ARG;
    OBM_CUDA(h, cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream_v;
    if (ndocs == 0) return OBM_OK;
    k_generate_corpus<<<(ndocs + 127) / 128, 128, 0, st>>>((uint8_t *)d_bytes, (uint64_t *)d_doc_off, ndocs, doc_bytes, first_doc, flavour);
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}


/* ------------------------------------------------------------------------------------------- */
/* SURVEY.md 8(f) rank 1 on the device: compact index of REGISTERED markers                    */
/* ------------------------------------------------------------------------------------------- */
/* One thread per document walks the document's tuples the way parser/state.go walks lexemes up to
 * loadDefinition (state.go:64-77, definition.go:13-21): MarkerStart "+" (Scope Separator)+ followed by an Arg,
 * with the joined name in the registry.  Emits one 16-byte record per such marker:
 *     { u32 doc, u32 tuple index inside the document, u32 offset of '+', u16 registry id, u16 scopes }
 * 8 markers x 16 B per 4 KiB manifest = 3 % of the input: this, not the 35 % tuple stream, is what ranks
 * exchange over NVLink (SURVEY section 7, hard part 1). */
struct DevRegistry { uint32_t n; uint32_t off[9]; uint8_t text[512]; }; /* names back to back, off[n] = end */

/* One WARP per document, a lane per tuple.  The document's tuples are staged in shared memory 256 at a time
 * (coalesced 8-byte loads) so the few MarkerStart candidates can look back for a stale buffer and forward along
 * the Scope/Separator chain without dependent global loads; the marker name is then compared with the registry
 * entries of the same length in one pass over the (contiguous) "+scope:scope" text, no early exit, so the byte
 * loads are independent.  Records keep tuple order (ballot ranks). */
constexpr uint32_t MI_STAGE = 256, MI_STEP = 192; /* tuples staged / tuples whose candidates are handled per round */
template <bool WRITE>
__global__ void __launch_bounds__(256)
k_marker_index(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, uint32_t ndocs,
               const obm_tuple *__restrict__ tuples, const uint64_t *__restrict__ tuple_off, DevRegistry reg,
               uint32_t *__restrict__ counts, const uint64_t *__restrict__ rec_off, uint4 *__restrict__ records, uint64_t cap) {
    __shared__ obm_tuple stage[8][MI_STAGE];
    obm_tuple *sm = stage[threadIdx.x >> 5];
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t d = warp; d < ndocs; d += nwarps) {
        const uint8_t *doc = bytes + doc_off[d];
        const obm_tuple *t = tuples + tuple_off[d];
        const uint32_t n = (uint32_t)(tuple_off[d + 1] - tuple_off[d]);
        uint32_t found = 0;
        uint64_t at = WRITE ? rec_off[d] : 0;
        for (uint32_t base = 0; base < n; base += MI_STEP) {
            /* stage [lo, lo + cnt): 32 tuples of look-back, the round's tuples, 32 of look-ahead */
            const uint32_t lo = base >= 32 ? base - 32 : 0, cnt = (n - lo < MI_STAGE) ? n - lo : MI_STAGE;
            __syncwarp();
            for (uint32_t k = lane; k < cnt; k += 32) sm[k] = t[lo + k];
            __syncwarp();
            auto T = [&](uint32_t j) -> obm_tuple { return (j >= lo && j - lo < cnt) ? sm[j - lo] : t[j]; };
            const uint32_t hi = (n - base < MI_STEP) ? n : base + MI_STEP;
            for (uint32_t c0 = base; c0 < hi; c0 += 32) {
                const uint32_t i = c0 + lane;
                const obm_tuple tu = i < hi ? T(i) : 0;
                int hit = -1; uint32_t scopes = 0;
                if (i < hi && OBM_TUPLE_KIND(tu) == OBM_K_MARKER_START && OBM_TUPLE_LEN(tu) == 1) {
                    /* the lexer's buffer must not hold stale text: walking back over tuples that carry no buffer text,
                     * the first PART / FLUSH / slice tuple decides */
                    bool clean = true;
                    for (uint32_t j = i; j-- > 0;) {
                        const uint32_t kj = OBM_TUPLE_KIND(T(j));
                        if (kj == OBM_K_PART) { clean = false; break; }
                        if (kj == OBM_K_FLUSH || (kj >= OBM_K_COMMENT && kj <= OBM_K_QUOTE)) break;
                    }
                    if (clean) {
                        /* "+scope:scope:...": Scope/Separator pairs tile the text after the '+', so the name is the
                         * contiguous slice doc[off, off + pos) */
                        uint32_t pos = 1, j = i + 1; bool contiguous = true;
                        const uint32_t off = OBM_TUPLE_OFF(tu);
                        for (;;) {
                            if (j + 1 >= n) break;
                            const obm_tuple a = T(j), b = T(j + 1);
                            if (OBM_TUPLE_KIND(a) != OBM_K_SCOPE || OBM_TUPLE_KIND(b) != OBM_K_SEPARATOR) break;
                            contiguous &= OBM_TUPLE_OFF(a) == off + pos + (scopes ? 1u : 0u);
                            pos += OBM_TUPLE_LEN(a) + (scopes ? 1u : 0u); scopes++; j += 2;
                        }
                        if (scopes && j < n && OBM_TUPLE_KIND(T(j)) == OBM_K_ARG) {
                            for (uint32_t r = 0; r < reg.n; r++) {
                                if (reg.off[r + 1] - reg.off[r] != pos) continue;
                                uint32_t diff = 0;
                                if (contiguous) {
                                    for (uint32_t b = 0; b < pos; b++) diff |= (uint32_t)doc[off + b] ^ (uint32_t)(uint8_t)reg.text[reg.off[r] + b];
                                } else { /* scope slices apart from each other: compare piece by piece */
                                    uint32_t q = 1; diff = (uint32_t)(uint8_t)reg.text[reg.off[r]] ^ (uint32_t)'+';
                                    for (uint32_t jj = i + 1, sc = 0; sc < scopes; jj += 2, sc++) {
                                        const obm_tuple a = T(jj);
                                        if (sc) { diff |= (uint32_t)(uint8_t)reg.text[reg.off[r] + q] ^ (uint32_t)':'; q++; }
                                        for (uint32_t b = 0; b < OBM_TUPLE_LEN(a); b++) diff |= (uint32_t)doc[OBM_TUPLE_OFF(a) + b] ^ (uint32_t)(uint8_t)reg.text[reg.off[r] + q + b];
                                        q += OBM_TUPLE_LEN(a);
                                    }
                                }
                                if (diff == 0) hit = (int)r;
                            }
                        }
                    }
                }
                const uint32_t bal = __ballot_sync(0xffffffffu, hit >= 0);
                if (WRITE && hit >= 0) {
                    const uint64_t w = at + (uint32_t)__popc(bal & ((1u << lane) - 1u));
                    if (w < cap) records[w] = make_uint4(d, i, OBM_TUPLE_OFF(tu), (uint32_t)hit | (scopes << 16));
                }
                at += (uint32_t)__popc(bal); found += (uint32_t)__popc(bal);
            }
        }
        if (!WRITE && lane == 0) counts[d] = found;
    }
}

extern "C" int obm_marker_index_device(obm_handle *h, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                                       const void *d_tuples, const void *d_doc_tuple_off, void *d_records, uint64_t cap,
                                       void *d_doc_rec_off, void *stream) {
    if (!h || !reg || !d_doc_off || !d_doc_tuple_off || !d_doc_rec_off) return OBM_E_ARG;
    OBM_CUDA(h, cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    DevRegistry R; memset(&R, 0, sizeof R);
    uint32_t nm = 0; const char *nmv[8]; uint32_t nml[8];
    nm = obm_registry_names(reg, nmv, nml, 8);
    if (obm_registry_names(reg, nullptr, nullptr, 0xFFFFFFFFu) > 8) { set_err(h, "the device index holds at most 8 marker names"); return OBM_E_ARG; }
    uint32_t o = 0;
    for (uint32_t r = 0; r < nm; r++) {
        if (o + nml[r] > sizeof R.text) { set_err(h, "registry too large for the device index"); return OBM_E_ARG; }
        R.off[r] = o; memcpy(R.text + o, nmv[r], nml[r]); o += nml[r];
    }
    R.off[nm] = o; R.n = nm;
    if (ndocs == 0) { OBM_CUDA(h, cudaMemsetAsync(d_doc_rec_off, 0, 8, st)); return OBM_OK; }
    uint64_t need = align_up((uint64_t)ndocs * 4 + 4, 256) + align_up((uint64_t)scan_tiles(ndocs) * 8 + 8, 256);
    if (h->scratch_bytes < need) {
        if (h->scratch) { OBM_CUDA(h, cudaStreamSynchronize(st)); cudaFree(h->scratch); h->scratch = nullptr; h->scratch_bytes = 0; }
        OBM_CUDA(h, cudaMalloc(&h->scratch, need)); h->scratch_bytes = need;
    }
    uint32_t *counts = (uint32_t *)h->scratch;
    uint64_t *tile_sums = (uint64_t *)((uint8_t *)h->scratch + align_up((uint64_t)ndocs * 4 + 4, 256));
    uint64_t *roff = (uint64_t *)d_doc_rec_off;
    int sms_i = 0;
    OBM_CUDA(h, cudaDeviceGetAttribute(&sms_i, cudaDevAttrMultiProcessorCount, h->device));
    const uint32_t nt = scan_tiles(ndocs);
    uint32_t nb = (uint32_t)sms_i * 8u; /* persistent warps, a document each per step */
    if (nb > (ndocs + 7) / 8) nb = (ndocs + 7) / 8;
    k_marker_index<false><<<nb, 256, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, (const obm_tuple *)d_tuples,
                                               (const uint64_t *)d_doc_tuple_off, R, counts, nullptr, nullptr, 0);
    k_scan_tiles<<<nt, SCAN_THREADS, 0, st>>>(counts, ndocs, roff, tile_sums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(tile_sums, nt, roff + ndocs);
    k_scan_add<<<nt, SCAN_THREADS, 0, st>>>(roff, ndocs, tile_sums, ~0ull, nullptr);
    if (d_records && cap)
        k_marker_index<true><<<nb, 256, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, (const obm_tuple *)d_tuples,
                                                  (const uint64_t *)d_doc_tuple_off, R, nullptr, roff, (uint4 *)d_records, cap);
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

/* ---- the same index, FLAT over the tuple stream (the exchange payload of the multi-GPU step) ----------------------------
 * k_marker_index above is a warp per document and spends its time on per-document bookkeeping.
 * Here a thread takes 8 consecutive tuples of the whole stream (four 16-byte loads, coalesced across the warp); the rare
 * MarkerStart candidates (4 % of the tuples) look around through the cache: back for a stale buffer, forward along the
 * Scope / Separator chain (a document's tuples end with EOF or a fatal error, so neither walk leaves the document), then the
 * name is compared with the registry.  One pass: tiles by ticket, the tile's hit count goes through a decoupled look-back
 * (obm_fast.cuh), the records are written in tuple order; the document of a hit is found from the tile's first tuple
 * (k_flat_tile_docs) in 64 cached offsets.  What bounds the kernel is the number of dependent round trips to memory per tile.  (Until round 2's last session: two passes and a bisection per hit.)  Records: {u32 doc + doc_base, u32 tuple index in the document, u32 offset of '+',
 * u16 registry id | u16 scopes << 16}. */
constexpr uint32_t FI_THREADS = 256, FI_PER = 8, FI_TILE = FI_THREADS * FI_PER;
/* the tuple stream as the candidate walks see it: the tile's own tuples from shared memory, the neighbours' from global memory */
struct TileView {
    const obm_tuple *g, *s; uint64_t t0;
    __device__ __forceinline__ obm_tuple operator[](uint64_t j) const { const uint64_t r = j - t0; return r < FI_TILE ? s[r] : g[j]; }
};
template <class TV>
__device__ __forceinline__ int flat_index_hit(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, uint32_t ndocs,
                                              const TV &t, const uint64_t *__restrict__ tuple_off, uint64_t ntup, uint64_t i,
                                              const DevRegistry &reg, uint32_t hint, bool exact, uint64_t exact_doc_off, uint32_t *doc_out, uint32_t *scopes_out) {
    const obm_tuple tu = t[i];
    /* stale buffer?  walk back over tuples that carry no buffer text; the first PART / FLUSH / slice tuple decides */
    for (uint64_t j = i; j-- > 0;) {
        const uint32_t kj = OBM_TUPLE_KIND(t[j]);
        if (kj == OBM_K_PART) return -1;
        if (kj == OBM_K_FLUSH || (kj >= OBM_K_COMMENT && kj <= OBM_K_QUOTE) || kj == OBM_K_EOF || kj >= OBM_K_ERR_MALFORMED) break;
    }
    uint32_t pos = 1, scopes = 0; uint64_t j = i + 1; bool contiguous = true;
    const uint32_t off = OBM_TUPLE_OFF(tu);
    for (;;) {
        if (j + 1 >= ntup) break;
        const obm_tuple a = t[j], b = t[j + 1];
        if (OBM_TUPLE_KIND(a) != OBM_K_SCOPE || OBM_TUPLE_KIND(b) != OBM_K_SEPARATOR) break;
        contiguous &= OBM_TUPLE_OFF(a) == off + pos + (scopes ? 1u : 0u);
        pos += OBM_TUPLE_LEN(a) + (scopes ? 1u : 0u); scopes++; j += 2;
    }
    if (!scopes || j >= ntup || OBM_TUPLE_KIND(t[j]) != OBM_K_ARG) return -1;
    bool len_ok = false;
    for (uint32_t r = 0; r < reg.n; r++) len_ok |= reg.off[r + 1] - reg.off[r] == pos;
    if (!len_ok) return -1;
    uint32_t lo = hint; /* last d with tuple_off[d] <= i; `exact`: the caller found it in its cached offsets, else walk on from the hint */
    if (!exact) while (lo + 1 < ndocs && tuple_off[lo + 1] <= i) lo++;
    const uint8_t *doc = bytes + (exact ? exact_doc_off : doc_off[lo]);
    int hit = -1;
    /* the usual case -- one contiguous name of at most 48 bytes -- with ONE round trip to the text: thirteen aligned words
     * loaded together, shifted into place, then compared byte by byte in registers (the byte loop below costs a round trip
     * per few bytes) */
    constexpr uint32_t NW = 12;
    uint32_t aw[NW];
    const bool vec = contiguous && pos <= 4 * NW;
    if (vec) {
        const uintptr_t p0 = (uintptr_t)(doc + off);
        const uint32_t *wp = reinterpret_cast<const uint32_t *>(p0 & ~(uintptr_t)3);
        const uint32_t sh = (uint32_t)(p0 & 3u) * 8u, need = ((uint32_t)(p0 & 3u) + pos + 3u) >> 2; /* words that hold the name */
        uint32_t w[NW + 1];
#pragma unroll
        for (uint32_t k = 0; k <= NW; k++) w[k] = k < need ? wp[k] : 0u;
#pragma unroll
        for (uint32_t k = 0; k < NW; k++) aw[k] = __funnelshift_r(w[k], w[k + 1], sh);
    }
    for (uint32_t r = 0; r < reg.n; r++) {
        if (reg.off[r + 1] - reg.off[r] != pos) continue;
        uint32_t diff = 0;
        if (vec) {
#pragma unroll
            for (uint32_t b = 0; b < 4 * NW; b++) if (b < pos) diff |= ((aw[b >> 2] >> (8u * (b & 3u))) & 0xFFu) ^ (uint32_t)(uint8_t)reg.text[reg.off[r] + b];
        } else if (contiguous) for (uint32_t b = 0; b < pos; b++) diff |= (uint32_t)doc[off + b] ^ (uint32_t)(uint8_t)reg.text[reg.off[r] + b];
        else { /* scope slices apart from each other: piece by piece */
            uint32_t q = 1; diff = (uint32_t)(uint8_t)reg.text[reg.off[r]] ^ (uint32_t)'+';
            uint64_t jj = i + 1;
            for (uint32_t sc = 0; sc < scopes; jj += 2, sc++) {
                const obm_tuple a = t[jj];
                if (sc) { diff |= (uint32_t)(uint8_t)reg.text[reg.off[r] + q] ^ (uint32_t)':'; q++; }
                for (uint32_t b = 0; b < OBM_TUPLE_LEN(a); b++) diff |= (uint32_t)doc[OBM_TUPLE_OFF(a) + b] ^ (uint32_t)(uint8_t)reg.text[reg.off[r] + q + b];
                q += OBM_TUPLE_LEN(a);
            }
        }
        if (diff == 0) hit = (int)r;
    }
    *doc_out = lo; *scopes_out = scopes;
    return hit;
}
/* tile -> the document of its first tuple: document d owns the tiles whose first tuple lies in [tuple_off[d], tuple_off[d + 1]) */
__global__ void __launch_bounds__(256)
k_flat_tile_docs(const uint64_t *__restrict__ tuple_off, uint32_t ndocs, uint32_t ntiles, uint32_t *__restrict__ tile_doc) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= ndocs) return;
    const uint64_t a = tuple_off[d], b = tuple_off[d + 1];
    for (uint64_t t = (a + FI_TILE - 1) / FI_TILE; t * FI_TILE < b && t < ntiles; t++) tile_doc[t] = d;
}
/* ONE pass: tiles by ticket.  The rare candidates are compacted (in tuple order) and then looked at a THREAD EACH -- the walks
 * around a candidate are a few hundred instructions, which single lanes of the loading warps would execute at 1/32 of the
 * issue rate --; the tile's records are staged in shared memory while its hit count goes through a decoupled look-back. */
constexpr uint32_t FI_DOCS = 64, FI_RECS = FI_TILE / 4 + 8; /* tuple offsets cached per tile; a hit is at least 4 tuples */
__global__ void __launch_bounds__(FI_THREADS, 6)
k_marker_index_flat(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, uint32_t ndocs, uint32_t doc_base,
                    const obm_tuple *__restrict__ tuples, const uint64_t *__restrict__ tuple_off, const __grid_constant__ DevRegistry reg,
                    volatile uint64_t *state, uint32_t *ticket, uint32_t ntiles, const uint32_t *__restrict__ tile_doc, uint64_t *__restrict__ total_out,
                    uint4 *__restrict__ records, uint64_t cap) {
    __shared__ uint32_t wsum[FI_THREADS / 32];
    __shared__ uint32_t s_tile;
    __shared__ uint64_t s_doff[FI_DOCS + 1];
    __shared__ uint64_t s_excl;
    __shared__ uint16_t cidx[FI_TILE];
    __shared__ uint64_t s_toff[FI_DOCS + 1];
    __shared__ uint4 recs[FI_RECS];
    __shared__ __align__(16) obm_tuple stup[FI_TILE]; /* the tile's tuples: the walks around a candidate stay on chip */
    if (threadIdx.x == 0) s_tile = atomicAdd(ticket, 1u);
    __syncthreads();
    const uint32_t tile = s_tile;
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t ntup = tuple_off[ndocs];
    const uint64_t t0 = (uint64_t)tile * FI_TILE, i0 = t0 + (uint64_t)threadIdx.x * FI_PER;
    uint32_t cand = 0;
    if (i0 + FI_PER <= ntup) { /* the stream is 8-byte aligned and i0 a multiple of 8 tuples: 64-byte chunks */
        const uint4 *p = reinterpret_cast<const uint4 *>(tuples + i0);
#pragma unroll
        for (uint32_t q = 0; q < FI_PER / 2; q++) {
            const uint4 x = p[q]; /* kind and length live in the high word */
            reinterpret_cast<uint4 *>(stup)[threadIdx.x * (FI_PER / 2) + q] = x;
            const obm_tuple a = (uint64_t)x.x | ((uint64_t)x.y << 32), b = (uint64_t)x.z | ((uint64_t)x.w << 32);
            if (OBM_TUPLE_KIND(a) == OBM_K_MARKER_START && OBM_TUPLE_LEN(a) == 1) cand |= 1u << (2 * q);
            if (OBM_TUPLE_KIND(b) == OBM_K_MARKER_START && OBM_TUPLE_LEN(b) == 1) cand |= 2u << (2 * q);
        }
    } else {
#pragma unroll
        for (uint32_t q = 0; q < FI_PER; q++) {
            const obm_tuple a = i0 + q < ntup ? tuples[i0 + q] : 0;
            stup[threadIdx.x * FI_PER + q] = a;
            if (i0 + q < ntup && OBM_TUPLE_KIND(a) == OBM_K_MARKER_START && OBM_TUPLE_LEN(a) == 1) cand |= 1u << q;
        }
    }
    /* the candidates of the tile, in tuple order */
    const uint32_t nc = (uint32_t)__popc(cand);
    uint32_t incl = nc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (uint32_t)o) incl += x; }
    if (lane == 31) wsum[wid] = incl;
    const uint32_t hint = t0 < ntup ? tile_doc[tile] : 0; /* the document of the tile's first tuple (k_flat_tile_docs) */
    __syncthreads();
    uint32_t cbase = incl - nc, ctot = 0;
#pragma unroll
    for (uint32_t w = 0; w < FI_THREADS / 32; w++) { const uint32_t c = wsum[w]; if (w < wid) cbase += c; ctot += c; }
    for (uint32_t m = cand; m; m &= m - 1) cidx[cbase++] = (uint16_t)(threadIdx.x * FI_PER + (uint32_t)__ffs((int)m) - 1u);
    if (ctot) for (uint32_t k = threadIdx.x; k <= 2 * FI_DOCS + 1; k += FI_THREADS) { /* ctot > 0 implies t0 < ntup */
        const uint32_t kk = k <= FI_DOCS ? k : k - FI_DOCS - 1;
        if (k <= FI_DOCS) s_toff[kk] = hint + kk <= ndocs ? tuple_off[hint + kk] : ~0ull;
        else s_doff[kk] = hint + kk <= ndocs ? doc_off[hint + kk] : 0;
    }
    __syncthreads();
    /* a thread per candidate, FI_THREADS per round; hits keep the order */
    uint32_t running = 0;
    for (uint32_t base = 0; base < ctot; base += FI_THREADS) { /* block-uniform */
        const uint32_t c = base + threadIdx.x;
        int hit = -1; uint4 rec = make_uint4(0, 0, 0, 0);
        if (c < ctot) {
            const uint64_t i = t0 + cidx[c];
            uint32_t lo = 0, hi = FI_DOCS + 1; /* last k with s_toff[k] <= i (s_toff[0] <= t0 <= i) */
            while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (s_toff[mid] <= i) lo = mid; else hi = mid; }
            uint32_t d = 0, scopes = 0;
            const TileView tv{tuples, stup, t0};
            hit = flat_index_hit(bytes, doc_off, ndocs, tv, tuple_off, ntup, i, reg, hint + lo, lo < FI_DOCS, s_doff[lo], &d, &scopes); /* lo == FI_DOCS: the cache ended, walk on */
            if (hit >= 0) rec = make_uint4(d + doc_base, (uint32_t)(i - (d - hint <= FI_DOCS ? s_toff[d - hint] : tuple_off[d])), OBM_TUPLE_OFF(tv[i]), (uint32_t)hit | (scopes << 16));
        }
        const uint32_t bal = __ballot_sync(0xffffffffu, hit >= 0);
        __syncthreads(); /* wsum of the previous use is read */
        if (lane == 0) wsum[wid] = (uint32_t)__popc(bal);
        __syncthreads();
        uint32_t pre = 0, tot = 0;
#pragma unroll
        for (uint32_t w = 0; w < FI_THREADS / 32; w++) { const uint32_t x = wsum[w]; if (w < wid) pre += x; tot += x; }
        const uint32_t at = running + pre + (uint32_t)__popc(bal & ((1u << lane) - 1u));
        if (hit >= 0 && at < FI_RECS) recs[at] = rec;
        running += tot;
    }
    if (wid == 0) {
        const uint64_t excl = obmf::lookback_warp(state, tile, running);
        if (lane == 0) { s_excl = excl; if (tile == ntiles - 1) *total_out = excl + running; }
    }
    __syncthreads();
    if (!records) return;
    const uint64_t at0 = s_excl;
    for (uint32_t k = threadIdx.x; k < running && k < FI_RECS; k += FI_THREADS) if (at0 + k < cap) records[at0 + k] = recs[k];
}

/* records of the REGISTERED markers of a resident tuple stream, in document order; *d_total (device u64) = their number.
 * Records beyond `cap` are not written.  doc_base is added to the document ids (global ids of a shard). */
extern "C" int obm_marker_index_flat_device(obm_handle *h, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, uint32_t doc_base,
                                            const void *d_tuples, const void *d_doc_tuple_off, uint64_t ntuples_bound, void *d_records, uint64_t cap,
                                            void *d_total, void *stream) {
    if (!h || !reg || !d_doc_off || !d_doc_tuple_off || !d_total) return OBM_E_ARG;
    OBM_CUDA(h, cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    DevRegistry R; memset(&R, 0, sizeof R);
    const char *nmv[8]; uint32_t nml[8];
    if (obm_registry_names(reg, nullptr, nullptr, 0xFFFFFFFFu) > 8) { set_err(h, "the device index holds at most 8 marker names"); return OBM_E_ARG; }
    const uint32_t nm = obm_registry_names(reg, nmv, nml, 8);
    uint32_t o = 0;
    for (uint32_t r = 0; r < nm; r++) {
        if (o + nml[r] > sizeof R.text) { set_err(h, "registry too large for the device index"); return OBM_E_ARG; }
        R.off[r] = o; memcpy(R.text + o, nmv[r], nml[r]); o += nml[r];
    }
    R.off[nm] = o; R.n = nm;
    if (ndocs == 0 || ntuples_bound == 0) { OBM_CUDA(h, cudaMemsetAsync(d_total, 0, 8, st)); return OBM_OK; }
    /* the tuple count lives on the device (doc_tuple_off[ndocs]); the grid is sized for the caller's bound (its out_cap) */
    const uint64_t ntiles64 = (ntuples_bound + FI_TILE - 1) / FI_TILE;
    if (ntiles64 > 0x7FFFFFF0ull) { set_err(h, "tuple stream too large for the flat index"); return OBM_E_ARG; }
    const uint32_t ntiles = (uint32_t)ntiles64;
    const uint64_t need = align_up((uint64_t)ntiles * 8, 256) + 256 + align_up((uint64_t)ntiles * 4, 256);
    if (h->scratch_bytes < need) {
        if (h->scratch) { OBM_CUDA(h, cudaStreamSynchronize(st)); cudaFree(h->scratch); h->scratch = nullptr; h->scratch_bytes = 0; }
        OBM_CUDA(h, cudaMalloc(&h->scratch, need)); h->scratch_bytes = need;
    }
    uint64_t *state = (uint64_t *)h->scratch;
    uint32_t *ticket = (uint32_t *)((uint8_t *)h->scratch + align_up((uint64_t)ntiles * 8, 256));
    uint32_t *tile_doc = (uint32_t *)((uint8_t *)ticket + 256);
    OBM_CUDA(h, cudaMemsetAsync(state, 0, need, st));
    k_flat_tile_docs<<<(ndocs + 255) / 256, 256, 0, st>>>((const uint64_t *)d_doc_tuple_off, ndocs, ntiles, tile_doc);
    k_marker_index_flat<<<ntiles, FI_THREADS, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, doc_base, (const obm_tuple *)d_tuples,
                                                      (const uint64_t *)d_doc_tuple_off, R, state, ticket, ntiles, tile_doc, (uint64_t *)d_total,
                                                      (d_records && cap) ? (uint4 *)d_records : nullptr, cap);
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

/* ------------------------------------------------------------------------------------------- */
/* SURVEY.md 8(f) rank 2: collection prefix rewrite (manifests/manifest.go:89-95) on the device  */
/* SURVEY.md 8(f) rank 4: manifest splitting on "---" lines (manifests/manifest.go:57-80)         */
/* One warp per document, two passes (count, exclusive scan, write)                              */
/* ------------------------------------------------------------------------------------------- */
__device__ __forceinline__ uint32_t eq_bytes4(uint32_t v, uint32_t pat) { /* 4-bit mask of bytes of v equal to pat's byte (exact for any byte value) */
    const uint32_t t = v ^ pat;
    const uint32_t z = ~(((t & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | t) & 0x80808080u;
    return ((z >> 7) * 0x00204081u >> 21) & 0xFu;
}
__device__ __forceinline__ bool dev_match(const uint8_t *p, uint32_t avail, const char *pat, uint32_t len) {
    if (avail < len) return false;
    for (uint32_t k = 0; k < len; k++) if (p[k] != (uint8_t)pat[k]) return false;
    return true;
}
/* strings.ReplaceAll(ReplaceAll(content, "+operator-builder:collection:field", "+operator-builder:field"),
 *                    "collectionField", "field"): the two patterns cannot overlap each other or themselves and the
 * first replacement cannot create an occurrence of the second, so one left-to-right pass is equivalent.  Both
 * replacements are deletions: "+operator-builder:" [collection:] "field" drops 11 bytes at +18, and
 * [collection] "Field" -> "field" drops 10 bytes and lowers one letter.
 *
 * One WARP per document.  Detection: 16 bytes per lane and step (aligned uint4), exact SIMD byte tests for '+'
 * and 'c', the rare candidates verified byte by byte.  Copy: the runs between deletions are moved with
 * byte-interleaved lanes (lane k moves bytes k, k+32, ...), so every load/store instruction touches one or two
 * sectors whatever the shift between input and output is. */
/* dst[0..len) = src[0..len) by one warp: up to 3 head bytes, then 4 destination-aligned bytes per lane and step
 * (two aligned source words funnel-shifted together when the source is not 4-aligned relative to the
 * destination; reads at most 2 bytes past the run -- inside the buffer slack obmarkers.h asks for), then the tail */
__device__ __forceinline__ void warp_copy_bytes(uint8_t *dst, const uint8_t *src, uint32_t len, uint32_t lane) {
    uint32_t head = (uint32_t)((4u - ((uintptr_t)dst & 3u)) & 3u);
    if (head > len) head = len;
    if (lane < head) dst[lane] = src[lane];
    dst += head; src += head; len -= head;
    const uint32_t nw = len >> 2, ms = (uint32_t)((uintptr_t)src & 3u);
    const uint32_t *sw = reinterpret_cast<const uint32_t *>(src - ms);
    uint32_t *dw = reinterpret_cast<uint32_t *>(dst);
    for (uint32_t j = lane; j < nw; j += 32) {
        const uint32_t a = sw[j], b = ms ? sw[j + 1] : 0u;
        dw[j] = __funnelshift_r(a, b, ms * 8u);
    }
    const uint32_t tail = len & 3u;
    if (lane < tail) dst[nw * 4 + lane] = src[nw * 4 + lane];
}
/* one document by one warp: rewritten into dst (WRITE); returns the rewritten length */
template <bool WRITE>
__device__ __forceinline__ uint32_t rewrite_doc_warp(const uint8_t *src, uint32_t n, uint8_t *dst, uint32_t lane) {
    const char P1[] = "+operator-builder:collection:field", P2[] = "collectionField";
    const uint32_t skew = (uint32_t)((uintptr_t)src & 15u);
    const uint4 *base = reinterpret_cast<const uint4 *>(src - skew);
    uint32_t cur = 0, o = 0; /* next input byte to copy, bytes written so far (warp-uniform) */
    for (uint32_t c0 = 0; c0 < n + skew; c0 += 512) {
        const uint32_t q0 = c0 + lane * 16u;
        uint32_t plus = 0, cee = 0;
        if (q0 < n + skew) {
            const uint4 v = base[q0 >> 4];
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int k = 0; k < 4; k++) { plus |= eq_bytes4(w[k], 0x2B2B2B2Bu) << (4 * k); cee |= eq_bytes4(w[k], 0x63636363u) << (4 * k); }
        }
        uint32_t keep = 0xFFFFu;
        if (q0 < skew) keep &= (skew - q0 >= 16) ? 0u : (0xFFFFu << (skew - q0));
        if (q0 + 16 > n + skew) keep &= (q0 >= n + skew) ? 0u : (0xFFFFu >> (q0 + 16 - n - skew));
        uint32_t m1 = 0, m2 = 0;
        for (uint32_t m = plus & keep; m; m &= m - 1) { const uint32_t b = (uint32_t)__ffs((int)m) - 1u, p = q0 + b - skew; if (dev_match(src + p, n - p, P1, 34)) m1 |= 1u << b; }
        for (uint32_t m = cee & keep; m; m &= m - 1) { const uint32_t b = (uint32_t)__ffs((int)m) - 1u, p = q0 + b - skew; if (dev_match(src + p, n - p, P2, 15)) m2 |= 1u << b; }
        /* matches of the step in position order; a "collectionField" inside an already deleted range cannot occur
         * (the deleted text is "collection:" / "collection") */
        uint32_t todo = __ballot_sync(0xffffffffu, (m1 | m2) != 0);
        while (todo) {
            const uint32_t owner = (uint32_t)__ffs((int)todo) - 1u;
            const uint32_t a1 = __shfl_sync(0xffffffffu, m1, owner), a2 = __shfl_sync(0xffffffffu, m2, owner);
            const uint32_t oq0 = c0 + owner * 16u;
            for (uint32_t m = a1 | a2; m; m &= m - 1) {
                const uint32_t b = (uint32_t)__ffs((int)m) - 1u, p = oq0 + b - skew;
                const bool first = (a1 >> b) & 1u;
                const uint32_t del0 = first ? p + 18 : p, del1 = first ? p + 29 : p + 10;
                if (del0 < cur) continue; /* defensive: never true for these two patterns */
                if (WRITE) {
                    warp_copy_bytes(dst + o, src + cur, del0 - cur, lane);
                    if (!first && lane == 0) dst[o + (del0 - cur)] = 'f'; /* "Field" -> "field": written after the run, before the next copy starts there */
                }
                o += del0 - cur; cur = del1;
                if (!first) { o += 1; cur += 1; } /* the lowered 'F' */
            }
            todo &= todo - 1;
        }
    }
    if (WRITE) warp_copy_bytes(dst + o, src + cur, n - cur, lane);
    o += n - cur;
    return o;
}

template <bool WRITE>
__global__ void __launch_bounds__(256)
k_rewrite_collection(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, uint32_t ndocs,
                     uint32_t *__restrict__ new_len, const uint64_t *__restrict__ new_off, uint8_t *__restrict__ out) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t d = warp; d < ndocs; d += nwarps) {
        const uint32_t o = rewrite_doc_warp<WRITE>(bytes + doc_off[d], (uint32_t)(doc_off[d + 1] - doc_off[d]), WRITE ? out + new_off[d] : nullptr, lane);
        if (!WRITE && lane == 0) new_len[d] = o;
    }
}

/* Each record: { u32 doc, u32 a, u32 b, u32 0 }: extracted manifest = "\n" + content[a:b) (ExtractManifests
 * rebuilds it as "\n" + line for every line between separators; a separator is a line that equals "---" after
 * trimming trailing spaces).  Lines between two separators form one record; so do the lines before the first
 * and after the last one (the final, possibly empty, line included).
 *
 * One WARP per document, 512 bytes per step: every lane loads 16 bytes (aligned uint4), builds a newline mask
 * and a dash mask with exact SIMD-within-register byte tests, and only the rare "dash at a line start" positions
 * are verified byte by byte.  Separators are then folded into records in order through warp-uniform state. */
template <bool WRITE>
__global__ void __launch_bounds__(256)
k_split_docs(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, uint32_t ndocs, uint32_t *__restrict__ counts,
             const uint64_t *__restrict__ rec_off, uint4 *__restrict__ records, uint64_t cap) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t d = warp; d < ndocs; d += nwarps) {
        const uint8_t *src = bytes + doc_off[d];
        const uint32_t n = (uint32_t)(doc_off[d + 1] - doc_off[d]);
        const uint32_t skew = (uint32_t)((uintptr_t)src & 15u);
        const uint4 *base = reinterpret_cast<const uint4 *>(src - skew);
        uint32_t found = 0;
        uint64_t at = WRITE ? rec_off[d] : 0;
        uint32_t rs = 0; bool closed = false; /* start of the open group; closed: the document ended with a separator */
        uint32_t prev_nl = 1;                   /* the byte before the document counts as a line end */
        for (uint32_t c0 = 0; c0 < n + skew; c0 += 512) {
            const uint32_t q0 = c0 + lane * 16u;            /* buffer-relative position of this lane's first byte */
            uint32_t nl = 0, da = 0;
            if (q0 < n + skew) {
                const uint4 v = base[q0 >> 4];
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int k = 0; k < 4; k++) { nl |= eq_bytes4(w[k], 0x0A0A0A0Au) << (4 * k); da |= eq_bytes4(w[k], 0x2D2D2D2Du) << (4 * k); }
            }
            /* keep document bytes only */
            uint32_t keep = 0xFFFFu;
            if (q0 < skew) keep &= (skew - q0 >= 16) ? 0u : (0xFFFFu << (skew - q0));
            if (q0 + 16 > n + skew) keep &= (q0 >= n + skew) ? 0u : (0xFFFFu >> (q0 + 16 - n - skew));
            nl &= keep; da &= keep;
            /* line starts: the byte after a newline, and the first byte of the document */
            uint32_t before = __shfl_up_sync(0xffffffffu, nl >> 15, 1);
            if (lane == 0) before = c0 == 0 ? 0u : prev_nl;
            uint32_t ls_mask = ((nl << 1) | (before & 1u)) & 0xFFFFu;
            if (q0 <= skew && skew < q0 + 16) ls_mask |= 1u << (skew - q0);
            prev_nl = __shfl_sync(0xffffffffu, nl >> 15, 31);
            uint32_t cand = da & ls_mask & keep;
            /* verify: "---" + spaces* + ('\n' | end) */
            uint32_t seps = 0;
            for (uint32_t m = cand; m; m &= m - 1) {
                const uint32_t b = (uint32_t)__ffs((int)m) - 1u, p = q0 + b - skew;
                if (p + 2 < n && src[p + 1] == '-' && src[p + 2] == '-') {
                    uint32_t e = p + 3;
                    while (e < n && src[e] == ' ') e++;
                    if (e == n || src[e] == '\n') seps |= 1u << b;
                }
            }
            /* fold the step's separators into records, in order */
            uint32_t todo = __ballot_sync(0xffffffffu, seps != 0);
            while (todo) {
                const uint32_t owner = (uint32_t)__ffs((int)todo) - 1u;
                uint32_t mine = __shfl_sync(0xffffffffu, seps, owner);
                const uint32_t oq0 = c0 + owner * 16u;
                while (mine) {
                    const uint32_t b = (uint32_t)__ffs((int)mine) - 1u; mine &= mine - 1;
                    const uint32_t ls = oq0 + b - skew;
                    uint32_t e = ls + 3;
                    while (e < n && src[e] == ' ') e++; /* every lane recomputes the (short) tail: warp-uniform */
                    if (rs < ls) { if (WRITE && lane == 0 && at < cap) records[at] = make_uint4(d, rs, ls - 1, 0); at++; found++; }
                    if (e < n) rs = e + 1; else closed = true;
                }
                todo &= todo - 1;
            }
        }
        if (!closed) { if (WRITE && lane == 0 && at < cap) records[at] = make_uint4(d, rs, n, 0); at++; found++; }
        if (!WRITE && lane == 0) counts[d] = found;
    }
}

static int two_pass_scratch(obm_handle *h, uint32_t ndocs, cudaStream_t st, uint32_t **counts, uint64_t **tile_sums) {
    uint64_t need = align_up((uint64_t)ndocs * 4 + 4, 256) + align_up((uint64_t)scan_tiles(ndocs) * 8 + 8, 256);
    if (h->scratch_bytes < need) {
        if (h->scratch) { OBM_CUDA(h, cudaStreamSynchronize(st)); cudaFree(h->scratch); h->scratch = nullptr; h->scratch_bytes = 0; }
        OBM_CUDA(h, cudaMalloc(&h->scratch, need)); h->scratch_bytes = need;
    }
    *counts = (uint32_t *)h->scratch;
    *tile_sums = (uint64_t *)((uint8_t *)h->scratch + align_up((uint64_t)ndocs * 4 + 4, 256));
    return OBM_OK;
}

/* ------------------------------------------------------------------------------------------- */
/* SURVEY.md 8(f) rank 1 proper: the parser on the device (csrc/obm_parse_dev.h), a thread per document */
/* ------------------------------------------------------------------------------------------- */
#include "obm_parse_dev.h"
extern "C" bool obm_registry_flatten(const obm_registry *r, obmr::DevTypedRegistry *D);
/* A thread per document, as many threads as the SM holds: the walk is a dependent chain of ~180 tuple reads per document,
 * i.e. latency-bound -- what hides the latency is the number of documents in flight, not staging (a version that staged 32
 * documents' tuples per warp in 48 KiB of shared memory ran at 4 warps per SM and was 11x slower). */
constexpr uint32_t PD_WARPS = 2, PD_CAP = 6144; /* k_hash_docs: warps per block; tuples staged per warp (48 KiB) */
/* TYPED: the registry holds a definition added with its Go struct type (obm_registry_define); the untyped walk takes the
 * registry without the type bytes, so its parameter block is the one it had before typing existed */
template <bool TYPED> using ParseRegistry = std::conditional_t<TYPED, obmr::DevTypedRegistry, obmr::DevRegistry>;
template <bool WRITE, bool TYPED>
__global__ void __launch_bounds__(128)
k_parse_docs(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, uint32_t ndocs, uint32_t doc_base,
             const obm_tuple *__restrict__ tuples, const uint64_t *__restrict__ tuple_off, const __grid_constant__ ParseRegistry<TYPED> R,
             uint32_t *__restrict__ cnt_res, uint32_t *__restrict__ cnt_args, const uint64_t *__restrict__ res_off, const uint64_t *__restrict__ arg_off,
             obm_result *__restrict__ res, uint64_t res_cap, obm_arg *__restrict__ args, uint64_t arg_cap) {
    const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= ndocs) return;
    const uint64_t t0 = tuple_off[d];
    obmr::Sink S{nullptr, 0, nullptr, 0, 0, 0, 0, 0};
    if (WRITE) { /* this document's slots: [res_off[d], res_off[d+1]) and [arg_off[d], arg_off[d+1]), clipped to the caller's capacity */
        S.res = res; S.args = args; S.res_at = res_off[d]; S.arg_at = arg_off[d];
        S.res_end = res_off[d + 1] < res_cap ? res_off[d + 1] : res_cap; S.arg_end = arg_off[d + 1] < arg_cap ? arg_off[d + 1] : arg_cap;
    }
    if constexpr (TYPED) {
        obmr::TypedSink TS; static_cast<obmr::Sink &>(TS) = S;
        obmr::parse_doc<true>(R, bytes + doc_off[d], tuples + t0, (uint32_t)(tuple_off[d + 1] - t0), d + doc_base, TS);
        S.nres = TS.nres; S.nargs = TS.nargs;
    } else obmr::parse_doc<false>(R, bytes + doc_off[d], tuples + t0, (uint32_t)(tuple_off[d + 1] - t0), d + doc_base, S);
    if (!WRITE) { cnt_res[d] = S.nres; cnt_args[d] = S.nargs; }
}

/* ------------------------------------------------------------------------------------------- */
/* per-document hash of the DECODED lexeme stream, on the device: the check BASELINE.md section 2 asks for at full size */
/* ------------------------------------------------------------------------------------------- */
/* FNV-1a (offset basis 0xcbf29ce484222325) over exactly the bytes obm_decode_doc / the oracle serialise per lexeme:
 * [u8 type][u32 line][u32 col][u32 vlen][value].  Walks plain lexemes and LINE tuples (Pos = {line, off - base + 1};
 * synthetic lexemes {0, 0} with values "true" / "\n" / ""); a document with pseudo-tuples the walk does not model or with
 * bytes >= 0x80 in a value (the decoder substitutes U+FFFD for invalid ones) gets hash 0 and counts in *n_host: hash those
 * on the host from obm_decode_doc.  Same staging as k_parse_docs: 32 documents' tuples per warp in shared memory. */
__device__ __forceinline__ uint64_t fnv1a_u8(uint64_t h, uint32_t b) { return (h ^ (uint64_t)b) * 0x100000001b3ull; }
__device__ __forceinline__ uint64_t fnv1a_u32(uint64_t h, uint32_t v) { h = fnv1a_u8(h, v & 0xFF); h = fnv1a_u8(h, (v >> 8) & 0xFF); h = fnv1a_u8(h, (v >> 16) & 0xFF); return fnv1a_u8(h, v >> 24); }
__global__ void __launch_bounds__(PD_WARPS * 32)
k_hash_docs(const uint8_t *__restrict__ bytes, const uint64_t *__restrict__ doc_off, uint32_t ndocs, const obm_tuple *__restrict__ tuples,
            const uint64_t *__restrict__ tuple_off, uint64_t *__restrict__ hashes, uint32_t *__restrict__ n_host) {
    extern __shared__ __align__(16) uint8_t pd_smem[];
    obm_tuple *sm = reinterpret_cast<obm_tuple *>(pd_smem) + (size_t)(threadIdx.x >> 5) * PD_CAP;
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t ngroups = (ndocs + 31) / 32;
    for (uint32_t g = blockIdx.x * PD_WARPS + (threadIdx.x >> 5); g < ngroups; g += gridDim.x * PD_WARPS) {
        const uint32_t dlo = g * 32, dhi = min(dlo + 32, ndocs);
        const uint64_t t_lo = tuple_off[dlo], t_hi = tuple_off[dhi];
        const bool staged = t_hi - t_lo <= PD_CAP;
        __syncwarp();
        if (staged) for (uint32_t k = lane; k < (uint32_t)(t_hi - t_lo); k += 32) sm[k] = tuples[t_lo + k];
        __syncwarp();
        const uint32_t d = dlo + lane;
        if (d >= dhi) continue;
        const uint64_t t0 = tuple_off[d];
        const obm_tuple *t = staged ? sm + (t0 - t_lo) : tuples + t0;
        const uint32_t nt = (uint32_t)(tuple_off[d + 1] - t0);
        const uint8_t *doc = bytes + doc_off[d];
        uint64_t h = 0xcbf29ce484222325ull;
        uint32_t line = 1, base = 0; bool host = false;
        for (uint32_t i = 0; i < nt && !host; i++) {
            const obm_tuple tu = t[i];
            const uint32_t k = OBM_TUPLE_KIND(tu), off = OBM_TUPLE_OFF(tu), len = OBM_TUPLE_LEN(tu);
            if (k == OBM_K_LINE) { base = off; line = len; continue; }
            if (k > OBM_K_EOF) { host = true; break; }
            const bool synthetic = k == OBM_K_SYNTHETIC_BOOL || k == OBM_K_MARKER_END || k == OBM_K_EOF;
            const uint32_t vlen = k == OBM_K_SYNTHETIC_BOOL ? 4u : k == OBM_K_MARKER_END ? 1u : k == OBM_K_EOF ? 0u : len;
            h = fnv1a_u8(h, k);
            h = fnv1a_u32(h, synthetic ? 0u : line);
            h = fnv1a_u32(h, synthetic ? 0u : off - base + 1u);
            h = fnv1a_u32(h, vlen);
            if (k == OBM_K_SYNTHETIC_BOOL) { h = fnv1a_u8(h, 't'); h = fnv1a_u8(h, 'r'); h = fnv1a_u8(h, 'u'); h = fnv1a_u8(h, 'e'); }
            else if (k == OBM_K_MARKER_END) h = fnv1a_u8(h, '\n');
            else if (k != OBM_K_EOF) for (uint32_t b = 0; b < len; b++) { const uint32_t c = doc[off + b]; if (c >= 0x80) host = true; h = fnv1a_u8(h, c); }
        }
        if (host) { atomicAdd(n_host, 1u); h = 0; }
        hashes[d] = h;
    }
}
extern "C" int obm_hash_batch_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, const void *d_tuples,
                                     const void *d_doc_tuple_off, void *d_hashes, void *d_n_host, void *stream) {
    if (!h || !d_doc_off || !d_doc_tuple_off || !d_hashes || !d_n_host) return OBM_E_ARG;
    OBM_CUDA(h, cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    OBM_CUDA(h, cudaMemsetAsync(d_n_host, 0, 4, st));
    if (ndocs == 0) return OBM_OK;
    const size_t pd_smem = (size_t)PD_WARPS * PD_CAP * sizeof(obm_tuple);
    OBM_CUDA(h, cudaFuncSetAttribute(k_hash_docs, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pd_smem));
    int sms_p = 0;
    OBM_CUDA(h, cudaDeviceGetAttribute(&sms_p, cudaDevAttrMultiProcessorCount, h->device));
    uint32_t nb = (uint32_t)sms_p * 2u;
    { const uint32_t gmax = ((ndocs + 31) / 32 + PD_WARPS - 1) / PD_WARPS; if (nb > gmax) nb = gmax; }
    k_hash_docs<<<nb, PD_WARPS * 32, pd_smem, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, (const obm_tuple *)d_tuples,
                                                   (const uint64_t *)d_doc_tuple_off, (uint64_t *)d_hashes, (uint32_t *)d_n_host);
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

/* obm_parse_batch_device on a flattened registry and the given scratch (the handle's, or a chunk slot's); *launches = kernels */
static int parse_device_impl(obm_handle *h, const obmr::DevTypedRegistry &R, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, uint32_t doc_base,
                             const void *d_tuples, const void *d_doc_tuple_off, void *d_results, uint64_t res_cap, void *d_args, uint64_t arg_cap,
                             void *d_doc_res_off, void *d_totals, cudaStream_t st, void **scratch_p, uint64_t *scratch_bytes_p, uint32_t *launches) {
    *launches = 0;
    uint64_t *roff = (uint64_t *)d_doc_res_off;
    if (ndocs == 0) { OBM_CUDA(h, cudaMemsetAsync(roff, 0, 8, st)); if (d_totals) OBM_CUDA(h, cudaMemsetAsync(d_totals, 0, 16, st)); return OBM_OK; }
    const uint64_t need = 2 * align_up((uint64_t)ndocs * 4 + 4, 256) + align_up(((uint64_t)ndocs + 1) * 8, 256) + align_up((uint64_t)scan_tiles(ndocs) * 8 + 8, 256);
    if (*scratch_bytes_p < need) {
        if (*scratch_p) { OBM_CUDA(h, cudaStreamSynchronize(st)); cudaFree(*scratch_p); *scratch_p = nullptr; *scratch_bytes_p = 0; }
        OBM_CUDA(h, cudaMalloc(scratch_p, need)); *scratch_bytes_p = need;
    }
    uint8_t *q = (uint8_t *)*scratch_p;
    uint32_t *cres = (uint32_t *)q; q += align_up((uint64_t)ndocs * 4 + 4, 256);
    uint32_t *carg = (uint32_t *)q; q += align_up((uint64_t)ndocs * 4 + 4, 256);
    uint64_t *aoff = (uint64_t *)q; q += align_up(((uint64_t)ndocs + 1) * 8, 256);
    uint64_t *tile_sums = (uint64_t *)q;
    const uint32_t nb = (ndocs + 127) / 128, nt = scan_tiles(ndocs);
    bool typed = false;
    for (uint32_t i = 0; i < R.n; i++) typed = typed || R.typed[i];
    const obmr::DevRegistry &RN = R; /* the untyped walk's parameter: the registry without its type bytes */
    if (typed)
        k_parse_docs<false, true><<<nb, 128, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, doc_base, (const obm_tuple *)d_tuples,
                                                      (const uint64_t *)d_doc_tuple_off, R, cres, carg, nullptr, nullptr, nullptr, 0, nullptr, 0);
    else
        k_parse_docs<false, false><<<nb, 128, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, doc_base, (const obm_tuple *)d_tuples,
                                                       (const uint64_t *)d_doc_tuple_off, RN, cres, carg, nullptr, nullptr, nullptr, 0, nullptr, 0);
    k_scan_tiles<<<nt, SCAN_THREADS, 0, st>>>(cres, ndocs, roff, tile_sums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(tile_sums, nt, roff + ndocs);
    k_scan_add<<<nt, SCAN_THREADS, 0, st>>>(roff, ndocs, tile_sums, ~0ull, nullptr);
    k_scan_tiles<<<nt, SCAN_THREADS, 0, st>>>(carg, ndocs, aoff, tile_sums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(tile_sums, nt, aoff + ndocs);
    k_scan_add<<<nt, SCAN_THREADS, 0, st>>>(aoff, ndocs, tile_sums, ~0ull, nullptr);
    if (d_totals) {
        OBM_CUDA(h, cudaMemcpyAsync(d_totals, roff + ndocs, 8, cudaMemcpyDeviceToDevice, st));
        OBM_CUDA(h, cudaMemcpyAsync((uint64_t *)d_totals + 1, aoff + ndocs, 8, cudaMemcpyDeviceToDevice, st));
    }
    if (d_results && d_args && typed)
        k_parse_docs<true, true><<<nb, 128, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, doc_base, (const obm_tuple *)d_tuples,
                                                     (const uint64_t *)d_doc_tuple_off, R, cres, carg, roff, aoff, (obm_result *)d_results, res_cap,
                                                     (obm_arg *)d_args, arg_cap);
    else if (d_results && d_args)
        k_parse_docs<true, false><<<nb, 128, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, doc_base, (const obm_tuple *)d_tuples,
                                                      (const uint64_t *)d_doc_tuple_off, RN, cres, carg, roff, aoff, (obm_result *)d_results, res_cap,
                                                      (obm_arg *)d_args, arg_cap);
    OBM_CUDA(h, cudaGetLastError());
    *launches = 7 + ((d_results && d_args) ? 1 : 0);
    return OBM_OK;
}

static bool flatten_for_device(obm_handle *h, const obm_registry *reg, obmr::DevTypedRegistry *R) {
    if (obm_registry_flatten(reg, R)) return true;
    set_err(h, "registry too large for the device parser (8 markers, 64 arguments, 1024 bytes of names)");
    return false;
}

extern "C" int obm_parse_batch_device(obm_handle *h, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, uint32_t doc_base,
                                      const void *d_tuples, const void *d_doc_tuple_off, void *d_results, uint64_t res_cap, void *d_args, uint64_t arg_cap,
                                      void *d_doc_res_off, void *d_totals, void *stream) {
    if (!h || !reg || !d_doc_off || !d_doc_tuple_off || !d_doc_res_off) return OBM_E_ARG;
    obmr::DevTypedRegistry R;
    if (!flatten_for_device(h, reg, &R)) return OBM_E_ARG;
    OBM_CUDA(h, cudaSetDevice(h->device));
    uint32_t launches;
    return parse_device_impl(h, R, d_bytes, d_doc_off, ndocs, doc_base, d_tuples, d_doc_tuple_off, d_results, res_cap, d_args, arg_cap, d_doc_res_off,
                             d_totals, (cudaStream_t)stream, &h->scratch, &h->scratch_bytes, &launches);
}

/* ------------------------------------------------------------------------------------------- */
/* obm_parse_batch: host batches through the slot pipeline of obm_lex_batch with the parser behind the scan; a chunk's   */
/* tuples stay on the device, only records, offsets and fallback tuples are copied back (obm_parse_gather.cuh)         */
/* ------------------------------------------------------------------------------------------- */
#include "obm_parse_gather.cuh"

struct ParseTotals { uint64_t res, args, host; uint32_t launches; };

static uint32_t grid_for(uint64_t items, uint32_t per_block) {
    const uint64_t g = (items + per_block - 1) / per_block;
    return (uint32_t)(g < 1 ? 1 : g > 8192 ? 8192 : g);
}

/* After the slot's scan: redo it while its result is unusable -- scratch overflow (the exact kernels, mode 1, as
 * obm_lex_batch does) or more tuples than the slot's buffer holds (grown to the count) -- then enqueue the parse, the
 * fallback gather and the D2H of the chunk's totals.  The record buffers are sized from the chunk's tuple count, which
 * bounds them: every Result and every argument belongs to a distinct tuple of its document (the walk writes one Result
 * per MarkerEnd, error or OBM_R_HOST tuple, one argument per value tuple), and fallback tuples are a subset. */
static int parse_chunk(obm_handle *h, obm_handle::Slot &sl, const obmr::DevTypedRegistry &R, ChunkTotals &T, ParseTotals &P) {
    const uint32_t nd = sl.d1 - sl.d0;
    const uint64_t nb = sl.h_doc_off[nd];
    int mode = h->mode, rc;
    for (;;) {
        OBM_CUDA(h, cudaEventSynchronize(sl.ev_scan));
        const uint32_t *stw = (const uint32_t *)&sl.h_info[1];
        if (stw[ST_RESERVED] && mode != 1) mode = 1;
        else if (sl.h_info[0] > sl.d_out_cap) { if ((rc = ensure(h, &sl.d_out, &sl.d_out_cap, sl.h_info[0])) != OBM_OK) return rc; }
        else break;
        const int saved = h->mode;
        h->mode = mode;
        rc = chunk_scan(h, sl, nb, true);
        h->mode = saved;
        if (rc != OBM_OK) return rc;
        P.launches += h->launches;
    }
    { float ms = 0.f; if (cudaEventElapsedTime(&ms, sl.ev_k0, sl.ev_k1) == cudaSuccess) T.ms_kernels += ms; }
    const uint32_t *stw = (const uint32_t *)&sl.h_info[1];
    const uint64_t ntup = sl.h_info[0];
    T.tuples += ntup; T.markers += sl.h_info[3]; T.lexemes += sl.h_info[4]; T.exact += stw[ST_DOCS_EXACT]; T.fatal += stw[ST_DOCS_FATAL];
    if ((rc = ensure(h, &sl.d_res, &sl.d_res_cap, ntup)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_args, &sl.d_args_cap, ntup)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_host, &sl.d_host_cap, ntup)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_res_off, &sl.d_res_off_cap, (uint64_t)nd + 1)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_host_off, &sl.d_host_off_cap, (uint64_t)nd + 1)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_host_cnt, &sl.d_host_cnt_cap, (uint64_t)nd + 1)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_host_sums, &sl.d_host_sums_cap, (uint64_t)scan_tiles(nd) + 1)) != OBM_OK) return rc;
    if ((rc = ensure(h, &sl.d_ptot, &sl.d_ptot_cap, 2)) != OBM_OK) return rc;
    OBM_CUDA(h, cudaEventRecord(sl.ev_k0, sl.st));
    uint32_t pl = 0;
    rc = parse_device_impl(h, R, sl.d_bytes, sl.d_doc_off, nd, sl.d0, sl.d_out, sl.d_tuple_off, sl.d_res, sl.d_res_cap, sl.d_args, sl.d_args_cap,
                           sl.d_res_off, sl.d_ptot, sl.st, &sl.scratch, &sl.scratch_bytes, &pl);
    if (rc != OBM_OK) return rc;
    const uint32_t nt = scan_tiles(nd);
    obmg::k_fallback_counts<<<grid_for(nd, obmg::THREADS), obmg::THREADS, 0, sl.st>>>(sl.d_res, sl.d_res_off, sl.d_tuple_off, nd, sl.d_host_cnt);
    k_scan_tiles<<<nt, SCAN_THREADS, 0, sl.st>>>(sl.d_host_cnt, nd, sl.d_host_off, sl.d_host_sums);
    k_scan_sums<<<1, SCAN_THREADS, 0, sl.st>>>(sl.d_host_sums, nt, sl.d_host_off + nd);
    k_scan_add<<<nt, SCAN_THREADS, 0, sl.st>>>(sl.d_host_off, nd, sl.d_host_sums, ~0ull, nullptr);
    obmg::k_fallback_gather<<<grid_for(nd, obmg::THREADS / 32), obmg::THREADS, 0, sl.st>>>(sl.d_out, sl.d_tuple_off, sl.d_host_off, nd, sl.d_host);
    OBM_CUDA(h, cudaGetLastError());
    P.launches += pl + 5;
    OBM_CUDA(h, cudaEventRecord(sl.ev_k1, sl.st));
    OBM_CUDA(h, cudaMemcpyAsync(&sl.h_info[5], sl.d_ptot, 16, cudaMemcpyDeviceToHost, sl.st));
    OBM_CUDA(h, cudaMemcpyAsync(&sl.h_info[7], sl.d_host_off + nd, 8, cudaMemcpyDeviceToHost, sl.st));
    OBM_CUDA(h, cudaEventRecord(sl.ev_scan, sl.st));
    return OBM_OK;
}

struct ParseOut {
    obm_result *results; uint64_t res_cap; obm_arg *args; uint64_t arg_cap; uint64_t *doc_res_off;
    obm_tuple *host_tuples; uint64_t host_cap; uint64_t *doc_host_off;
};

/* wait for the slot's parse, rebase its records and offsets by the totals of the chunks before it, and enqueue their D2H
 * at the final host positions; an array whose running total passes its capacity is not copied from there on */
static int parse_retire(obm_handle *h, obm_handle::Slot &sl, const ParseOut &O, ChunkTotals &T, ParseTotals &P) {
    OBM_CUDA(h, cudaEventSynchronize(sl.ev_scan));
    { float ms = 0.f; if (cudaEventElapsedTime(&ms, sl.ev_k0, sl.ev_k1) == cudaSuccess) T.ms_kernels += ms; }
    const uint32_t nd = sl.d1 - sl.d0;
    const uint64_t nres = sl.h_info[5], nargs = sl.h_info[6], nhost = sl.h_info[7];
    if (P.res || P.args || P.host) {
        obmg::k_rebase_records<<<grid_for(nres > nd ? nres : nd, obmg::THREADS), obmg::THREADS, 0, sl.st>>>(
            sl.d_res, nres, (uint32_t)P.args, sl.d_res_off, P.res, sl.d_host_off, P.host, nd);
        OBM_CUDA(h, cudaGetLastError());
        P.launches += 1;
    }
    OBM_CUDA(h, cudaMemcpyAsync(O.doc_res_off + sl.d0, sl.d_res_off, (uint64_t)nd * 8, cudaMemcpyDeviceToHost, sl.st));
    OBM_CUDA(h, cudaMemcpyAsync(O.doc_host_off + sl.d0, sl.d_host_off, (uint64_t)nd * 8, cudaMemcpyDeviceToHost, sl.st));
    if (O.results && nres && P.res + nres <= O.res_cap)
        OBM_CUDA(h, cudaMemcpyAsync(O.results + P.res, sl.d_res, nres * sizeof(obm_result), cudaMemcpyDeviceToHost, sl.st));
    if (O.args && nargs && P.args + nargs <= O.arg_cap)
        OBM_CUDA(h, cudaMemcpyAsync(O.args + P.args, sl.d_args, nargs * sizeof(obm_arg), cudaMemcpyDeviceToHost, sl.st));
    if (O.host_tuples && nhost && P.host + nhost <= O.host_cap)
        OBM_CUDA(h, cudaMemcpyAsync(O.host_tuples + P.host, sl.d_host, nhost * sizeof(obm_tuple), cudaMemcpyDeviceToHost, sl.st));
    P.res += nres; P.args += nargs; P.host += nhost;
    sl.busy = false;
    return OBM_OK;
}

extern "C" int obm_parse_batch(obm_handle *h, const obm_registry *reg, const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs,
                               obm_result *results, uint64_t res_cap, obm_arg *args, uint64_t arg_cap, uint64_t *doc_res_off,
                               obm_tuple *host_tuples, uint64_t host_cap, uint64_t *doc_host_off, uint64_t *totals, obm_stats *stats) {
    if (!h) return OBM_E_ARG;
    if (!reg || !doc_off || !doc_res_off || !doc_host_off || !totals) {
        set_err(h, "reg, doc_off, doc_res_off, doc_host_off and totals must not be NULL"); return OBM_E_ARG;
    }
    int rc;
    if ((rc = check_host_batch(h, bytes, doc_off, ndocs)) != OBM_OK) return rc;
    obmr::DevTypedRegistry R;
    if (!flatten_for_device(h, reg, &R)) return OBM_E_ARG;
    OBM_CUDA(h, cudaSetDevice(h->device));
    if ((rc = slots_init(h)) != OBM_OK) return rc;
    const ParseOut O{results, results ? res_cap : 0, args, args ? arg_cap : 0, doc_res_off, host_tuples, host_tuples ? host_cap : 0, doc_host_off};
    const uint64_t total = doc_off[ndocs] - doc_off[0];
    OBM_CUDA(h, cudaEventRecord(h->ev[0], h->stream));
    /* a batch of fewer than two chunks is one chunk: the same code path, without the overlap */
    const bool one = total < 2 * h->chunk_bytes || ndocs < 4;
    uint32_t nck = 0;
    Ck *cks = cut_chunks(doc_off, ndocs, one ? total + 1 : h->chunk_bytes, &nck);
    if (!cks) return OBM_E_NOMEM;
    ChunkTotals T = {0, 0, 0, 0, 0, false, false, 0.f};
    ParseTotals P = {0, 0, 0, 0};
    int err = OBM_OK;
    /* iteration k: issue chunk k (H2D + scan), parse chunk k-1, retire chunk k-2 */
    for (uint32_t k = 0; k < nck + 2 && err == OBM_OK; k++) {
        if (k < nck) {
            obm_handle::Slot &sl = h->slots[k % 3];
            if (k >= 3) { cudaError_t e_ = cudaStreamSynchronize(sl.st); if (e_ != cudaSuccess) { set_err(h, "cudaStreamSynchronize failed: %s", cudaGetErrorString(e_)); err = OBM_E_CUDA; break; } }
            if ((err = chunk_issue(h, sl, bytes, doc_off, cks[k].d0, cks[k].d1, true)) != OBM_OK) break;
            P.launches += h->launches;
        }
        if (k >= 1 && k - 1 < nck && (err = parse_chunk(h, h->slots[(k - 1) % 3], R, T, P)) != OBM_OK) break;
        if (k >= 2 && k - 2 < nck) err = parse_retire(h, h->slots[(k - 2) % 3], O, T, P);
    }
    for (auto &sl : h->slots) cudaStreamSynchronize(sl.st);
    free(cks);
    if (err != OBM_OK) return err;
    doc_res_off[ndocs] = P.res; doc_host_off[ndocs] = P.host;
    totals[0] = P.res; totals[1] = P.args; totals[2] = P.host;
    h->launches = P.launches;
    int result = OBM_OK;
    if (P.res > O.res_cap || P.args > O.arg_cap || P.host > O.host_cap) {
        set_err(h, "capacity too small: %llu results (cap %llu), %llu args (cap %llu), %llu fallback tuples (cap %llu)",
                (unsigned long long)P.res, (unsigned long long)O.res_cap, (unsigned long long)P.args, (unsigned long long)O.arg_cap,
                (unsigned long long)P.host, (unsigned long long)O.host_cap);
        result = OBM_E_CAPACITY;
    }
    OBM_CUDA(h, cudaEventRecord(h->ev[3], h->stream));
    OBM_CUDA(h, cudaStreamSynchronize(h->stream));
    if (stats) {
        memset(stats, 0, sizeof *stats);
        stats->n_tuples = T.tuples; stats->n_markers = T.markers; stats->n_lexemes = T.lexemes;
        stats->n_docs_exact = T.exact; stats->n_docs_fatal = T.fatal; stats->bytes = total;
        cudaEventElapsedTime(&stats->ms_total, h->ev[0], h->ev[3]);
        stats->ms_kernels = T.ms_kernels; /* scan + parse + gather, summed over the chunks */
    }
    return result;
}

#include "obm_rewrite.cuh"
/* one pass (obm_rewrite.cuh) when both buffers are 16-byte aligned, else r01's two passes over the documents */
extern "C" int obm_rewrite_collection_markers_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                                                     void *d_out_bytes, uint64_t out_cap, void *d_out_doc_off, void *stream) {
    if (!h || !d_doc_off || !d_out_doc_off) return OBM_E_ARG;
    OBM_CUDA(h, cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (ndocs == 0) { OBM_CUDA(h, cudaMemsetAsync(d_out_doc_off, 0, 8, st)); return OBM_OK; }
    uint64_t *noff = (uint64_t *)d_out_doc_off;
    int sms_i = 0;
    OBM_CUDA(h, cudaDeviceGetAttribute(&sms_i, cudaDevAttrMultiProcessorCount, h->device));
    const bool aligned = (((uintptr_t)d_bytes | (uintptr_t)d_out_bytes) & 15u) == 0;
    if (aligned && !getenv("OBM_REWRITE_TWO_PASS")) {
        uint64_t total = 0; /* the batch size: the last offset (8 bytes from the device; the call is synchronous at its end anyway) */
        OBM_CUDA(h, cudaMemcpyAsync(&total, (const uint64_t *)d_doc_off + ndocs, 8, cudaMemcpyDeviceToHost, st));
        OBM_CUDA(h, cudaStreamSynchronize(st));
        const uint64_t nch64 = total / obmrw::RW_CH + 1;
        if (nch64 > 0xFFFFFFF0ull) { set_err(h, "batch too large for the chunk index"); return OBM_E_ARG; }
        const uint32_t nchunks = (uint32_t)nch64;
        const uint64_t need = align_up(((uint64_t)nchunks + 2) * 4, 256) + align_up((uint64_t)nchunks * 8, 256) + 256;
        if (h->scratch_bytes < need) {
            if (h->scratch) { OBM_CUDA(h, cudaStreamSynchronize(st)); cudaFree(h->scratch); h->scratch = nullptr; h->scratch_bytes = 0; }
            OBM_CUDA(h, cudaMalloc(&h->scratch, need)); h->scratch_bytes = need;
        }
        uint32_t *tile_first = (uint32_t *)h->scratch;
        uint64_t *state = (uint64_t *)((uint8_t *)h->scratch + align_up(((uint64_t)nchunks + 2) * 4, 256));
        uint32_t *ticket = (uint32_t *)((uint8_t *)state + align_up((uint64_t)nchunks * 8, 256));
        OBM_CUDA(h, cudaMemsetAsync(state, 0, align_up((uint64_t)nchunks * 8, 256) + 256, st));
        obmrw::k_rw_tile_index<<<(ndocs + 1 + 255) / 256, 256, 0, st>>>((const uint64_t *)d_doc_off, ndocs, nchunks, tile_first);
        uint32_t nb = (uint32_t)sms_i * 8u; /* persistent CTAs, chunks by ticket */
        if (nb > nchunks) nb = nchunks;
        if (d_out_bytes)
            obmrw::k_rw_chunks<true><<<nb, obmrw::RW_THREADS, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, total, nchunks, tile_first,
                                                                        state, ticket, noff, (uint8_t *)d_out_bytes, out_cap);
        else
            obmrw::k_rw_chunks<false><<<nb, obmrw::RW_THREADS, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, total, nchunks, tile_first,
                                                                         state, ticket, noff, nullptr, 0);
        OBM_CUDA(h, cudaGetLastError());
        if (d_out_bytes) { /* the kernel never writes past out_cap; tell the caller when that cut the output short */
            uint64_t nt = 0;
            OBM_CUDA(h, cudaMemcpyAsync(&nt, noff + ndocs, 8, cudaMemcpyDeviceToHost, st));
            OBM_CUDA(h, cudaStreamSynchronize(st));
            if (nt > out_cap) { set_err(h, "rewrite needs %llu bytes, out_cap is %llu", (unsigned long long)nt, (unsigned long long)out_cap); return OBM_E_CAPACITY; }
        }
        return OBM_OK;
    }
    uint32_t *counts; uint64_t *tile_sums; int rc;
    if ((rc = two_pass_scratch(h, ndocs, st, &counts, &tile_sums)) != OBM_OK) return rc;
    const uint32_t nt = scan_tiles(ndocs);
    uint32_t nb = (uint32_t)sms_i * 8u; /* persistent warps, a document each per step */
    if (nb > (ndocs + 7) / 8) nb = (ndocs + 7) / 8;
    k_rewrite_collection<false><<<nb, 256, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, counts, nullptr, nullptr);
    k_scan_tiles<<<nt, SCAN_THREADS, 0, st>>>(counts, ndocs, noff, tile_sums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(tile_sums, nt, noff + ndocs);
    k_scan_add<<<nt, SCAN_THREADS, 0, st>>>(noff, ndocs, tile_sums, ~0ull, nullptr);
    if (d_out_bytes) { /* the rewritten size is known now: never write past the caller's buffer */
        uint64_t total = 0;
        OBM_CUDA(h, cudaMemcpyAsync(&total, noff + ndocs, 8, cudaMemcpyDeviceToHost, st));
        OBM_CUDA(h, cudaStreamSynchronize(st));
        if (total > out_cap) { set_err(h, "rewrite needs %llu bytes, out_cap is %llu", (unsigned long long)total, (unsigned long long)out_cap); return OBM_E_CAPACITY; }
    }
    if (d_out_bytes)
        k_rewrite_collection<true><<<nb, 256, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, nullptr, noff, (uint8_t *)d_out_bytes);
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

/* Manifest.LoadContent's collection rewrite and the scan of its result: obm_rewrite_collection_markers_device, then
 * obm_lex_batch_device over the rewritten batch (in the handle's mode).  Synchronous: the scan is sized by the
 * rewritten total, read back from the device. */
extern "C" int obm_lex_collection_batch_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, uint64_t total_bytes,
                                               void *d_out_bytes, uint64_t out_bytes_cap, void *d_out_doc_off, void *d_out, uint64_t out_cap,
                                               void *d_doc_tuple_off, void *d_status, void *d_counts, void *stream) {
    if (!h) return OBM_E_ARG;
    if (!d_out_doc_off || (total_bytes && !d_out_bytes)) { set_err(h, "null device pointer"); return OBM_E_ARG; }
    if (out_bytes_cap < total_bytes) {
        set_err(h, "out_bytes_cap %llu < total_bytes %llu (the rewrite never lengthens the text)", (unsigned long long)out_bytes_cap, (unsigned long long)total_bytes);
        return OBM_E_ARG;
    }
    if ((uintptr_t)d_out_bytes & 15u) { set_err(h, "d_out_bytes must be 16-byte aligned"); return OBM_E_ARG; }
    const uintptr_t in0 = (uintptr_t)d_bytes, out0 = (uintptr_t)d_out_bytes;
    if (total_bytes && in0 < out0 + out_bytes_cap && out0 < in0 + total_bytes) { set_err(h, "d_out_bytes overlaps d_bytes"); return OBM_E_ARG; }
    cudaStream_t st = (cudaStream_t)stream;
    int rc = obm_rewrite_collection_markers_device(h, d_bytes, d_doc_off, ndocs, d_out_bytes, out_bytes_cap, d_out_doc_off, stream);
    if (rc != OBM_OK) return rc;
    uint64_t rewritten = 0;
    if (ndocs) {
        OBM_CUDA(h, cudaMemcpyAsync(&rewritten, (const uint64_t *)d_out_doc_off + ndocs, 8, cudaMemcpyDeviceToHost, st));
        OBM_CUDA(h, cudaStreamSynchronize(st));
    }
    return obm_lex_batch_device(h, d_out_bytes, d_out_doc_off, ndocs, rewritten, d_out, out_cap, d_doc_tuple_off, d_status, d_counts, stream);
}

extern "C" int obm_split_docs_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, void *d_records, uint64_t cap,
                                     void *d_doc_rec_off, void *stream) {
    if (!h || !d_doc_off || !d_doc_rec_off) return OBM_E_ARG;
    OBM_CUDA(h, cudaSetDevice(h->device));
    cudaStream_t st = (cudaStream_t)stream;
    if (ndocs == 0) { OBM_CUDA(h, cudaMemsetAsync(d_doc_rec_off, 0, 8, st)); return OBM_OK; }
    uint32_t *counts; uint64_t *tile_sums; int rc;
    if ((rc = two_pass_scratch(h, ndocs, st, &counts, &tile_sums)) != OBM_OK) return rc;
    uint64_t *roff = (uint64_t *)d_doc_rec_off;
    int sms_i = 0;
    OBM_CUDA(h, cudaDeviceGetAttribute(&sms_i, cudaDevAttrMultiProcessorCount, h->device));
    const uint32_t nt = scan_tiles(ndocs);
    uint32_t nb = (uint32_t)sms_i * 8u; /* persistent warps, a document each per step */
    if (nb > (ndocs + 7) / 8) nb = (ndocs + 7) / 8;
    k_split_docs<false><<<nb, 256, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, counts, nullptr, nullptr, 0);
    k_scan_tiles<<<nt, SCAN_THREADS, 0, st>>>(counts, ndocs, roff, tile_sums);
    k_scan_sums<<<1, SCAN_THREADS, 0, st>>>(tile_sums, nt, roff + ndocs);
    k_scan_add<<<nt, SCAN_THREADS, 0, st>>>(roff, ndocs, tile_sums, ~0ull, nullptr);
    if (d_records && cap)
        k_split_docs<true><<<nb, 256, 0, st>>>((const uint8_t *)d_bytes, (const uint64_t *)d_doc_off, ndocs, nullptr, roff, (uint4 *)d_records, cap);
    OBM_CUDA(h, cudaGetLastError());
    return OBM_OK;
}

/* ------------------------------------------------------------------------------------------- */
/* multi-GPU: one rank per GPU, one NCCL all-gather of the Result records (SURVEY.md 8(b), 8(e))  */
/* ------------------------------------------------------------------------------------------- */
/* NCCL is bound at run time so that libobmarkers.so loads (and the single-GPU path works) on a box without it */
namespace {
typedef struct ncclComm *ncclComm_t;
struct NcclUniqueId { char internal[128]; };
struct NcclApi {
    void *lib;
    int (*GetUniqueId)(NcclUniqueId *);
    int (*CommInitRank)(ncclComm_t *, int, NcclUniqueId, int);
    int (*CommDestroy)(ncclComm_t);
    int (*AllGather)(const void *, void *, size_t, int /* ncclDataType_t */, ncclComm_t, cudaStream_t);
    const char *(*GetErrorString)(int);
};
NcclApi *nccl_api() {
    static NcclApi api; static int state = 0; /* 0 untried, 1 ok, -1 failed */
    if (state == 0) {
        const char *names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char *n : names) { api.lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (api.lib) break; }
        state = -1;
        if (api.lib) {
            api.GetUniqueId = (int (*)(NcclUniqueId *))dlsym(api.lib, "ncclGetUniqueId");
            api.CommInitRank = (int (*)(ncclComm_t *, int, NcclUniqueId, int))dlsym(api.lib, "ncclCommInitRank");
            api.CommDestroy = (int (*)(ncclComm_t))dlsym(api.lib, "ncclCommDestroy");
            api.AllGather = (int (*)(const void *, void *, size_t, int, ncclComm_t, cudaStream_t))dlsym(api.lib, "ncclAllGather");
            api.GetErrorString = (const char *(*)(int))dlsym(api.lib, "ncclGetErrorString");
            if (api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.GetErrorString) state = 1;
        }
    }
    return state == 1 ? &api : nullptr;
}
constexpr int NCCL_UINT8 = 1, NCCL_UINT64 = 5; /* ncclDataType_t: ncclUint8 = 1, ncclUint64 = 5 (nccl.h) */
}
struct obm_comm {
    obm_handle *h; ncclComm_t comm; int rank, nranks;
    uint64_t *d_counts_all; uint64_t *h_counts; /* [nranks]: device / pinned host */
    uint64_t *d_totals;                        /* {results, args} of the last step */
};
#define OBM_NCCL(h, call)                                                                                 \
    do { int e_ = (call); if (e_ != 0) { set_err((h), "%s failed: %s", #call, nccl_api()->GetErrorString(e_)); return OBM_E_CUDA; } } while (0)

extern "C" int obm_comm_unique_id(uint8_t *id) {
    NcclApi *N = nccl_api();
    if (!id) return OBM_E_ARG;
    if (!N) { set_err(nullptr, "libnccl.so.2 not found: the multi-GPU entry points need NCCL"); return OBM_E_NO_DEVICE; }
    NcclUniqueId u;
    if (N->GetUniqueId(&u) != 0) { set_err(nullptr, "ncclGetUniqueId failed"); return OBM_E_CUDA; }
    memcpy(id, u.internal, OBM_COMM_ID_BYTES);
    return OBM_OK;
}
extern "C" int obm_comm_create(obm_handle *h, const uint8_t *id, int rank, int nranks, obm_comm **out) {
    if (!h || !id || !out || nranks < 1 || rank < 0 || rank >= nranks) return OBM_E_ARG;
    *out = nullptr;
    NcclApi *N = nccl_api();
    if (!N) { set_err(h, "libnccl.so.2 not found: the multi-GPU entry points need NCCL"); return OBM_E_NO_DEVICE; }
    OBM_CUDA(h, cudaSetDevice(h->device));
    obm_comm *c = new (std::nothrow) obm_comm();
    if (!c) return OBM_E_NOMEM;
    memset(c, 0, sizeof *c);
    c->h = h; c->rank = rank; c->nranks = nranks;
    NcclUniqueId u; memcpy(u.internal, id, OBM_COMM_ID_BYTES);
    int e = N->CommInitRank(&c->comm, nranks, u, rank);
    if (e != 0) { set_err(h, "ncclCommInitRank failed: %s", N->GetErrorString(e)); delete c; return OBM_E_CUDA; }
    if (cudaMalloc(&c->d_counts_all, (size_t)nranks * 8) != cudaSuccess || cudaMalloc(&c->d_totals, 16) != cudaSuccess ||
        cudaHostAlloc((void **)&c->h_counts, (size_t)nranks * 8, cudaHostAllocDefault) != cudaSuccess) {
        set_err(h, "obm_comm_create: allocation failed"); N->CommDestroy(c->comm); delete c; return OBM_E_CUDA;
    }
    *out = c;
    return OBM_OK;
}
extern "C" void obm_comm_destroy(obm_comm *c) {
    if (!c) return;
    cudaSetDevice(c->h->device);
    if (nccl_api()) nccl_api()->CommDestroy(c->comm);
    cudaFree(c->d_counts_all); cudaFree(c->d_totals); cudaFreeHost(c->h_counts);
    delete c;
}
extern "C" int obm_marker_index_flat_device(obm_handle *h, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, uint32_t doc_base,
                                            const void *d_tuples, const void *d_doc_tuple_off, uint64_t ntuples_bound, void *d_records, uint64_t cap,
                                            void *d_total, void *stream);
extern "C" int obm_lex_batch_sharded_device(obm_comm *c, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                                            uint64_t total_bytes, uint32_t first_doc, void *d_out, uint64_t out_cap, void *d_doc_tuple_off, void *d_status,
                                            void *d_counts, void *d_index, uint64_t index_cap, void *d_index_all, uint64_t index_all_cap,
                                            uint64_t *rank_records, uint64_t *stride, void *stream) {
    if (!c || !reg || !d_out || !d_index || !d_index_all || !rank_records || !stride) return OBM_E_ARG;
    obm_handle *h = c->h; NcclApi *N = nccl_api(); cudaStream_t st = (cudaStream_t)stream;
    int rc = obm_lex_batch_device(h, d_bytes, d_doc_off, ndocs, total_bytes, d_out, out_cap, d_doc_tuple_off, d_status, d_counts, stream);
    if (rc != OBM_OK) return rc;
    rc = obm_marker_index_flat_device(h, reg, d_bytes, d_doc_off, ndocs, first_doc, d_out, d_doc_tuple_off, out_cap, d_index, index_cap, c->d_totals, stream);
    if (rc != OBM_OK) return rc;
    /* how many records does every rank hold?  (8 bytes per rank; the host needs the largest to size the slots) */
    OBM_NCCL(h, N->AllGather(c->d_totals, c->d_counts_all, 1, NCCL_UINT64, c->comm, st));
    OBM_CUDA(h, cudaMemcpyAsync(c->h_counts, c->d_counts_all, (size_t)c->nranks * 8, cudaMemcpyDeviceToHost, st));
    OBM_CUDA(h, cudaStreamSynchronize(st));
    uint64_t mx = 0;
    for (int r = 0; r < c->nranks; r++) { rank_records[r] = c->h_counts[r]; if (c->h_counts[r] > mx) mx = c->h_counts[r]; }
    *stride = mx;
    if (mx > index_cap || mx * (uint64_t)c->nranks > index_all_cap) {
        set_err(h, "index capacity: need %llu records per rank (send buffer and slot) and %llu in all", (unsigned long long)mx, (unsigned long long)(mx * c->nranks));
        return OBM_E_CAPACITY;
    }
    if (mx) OBM_NCCL(h, N->AllGather(d_index, d_index_all, (size_t)mx * 16, NCCL_UINT8, c->comm, st));
    return OBM_OK;
}

/* Host copy of the same generator (test/bench utility; no lexing). */
extern "C" int obm_generate_corpus_host(uint8_t *bytes, uint64_t *doc_off, uint32_t ndocs, uint32_t doc_bytes,
                                        uint64_t first_doc, int flavour) {
    if (!bytes) return OBM_E_ARG;
    for (uint32_t d = 0; d < ndocs; d++) {
        if (doc_off) doc_off[d] = (uint64_t)d * doc_bytes;
        obmc::generate_doc(bytes + (uint64_t)d * doc_bytes, doc_bytes, first_doc + d, flavour);
    }
    if (doc_off) doc_off[ndocs] = (uint64_t)ndocs * doc_bytes;
    return OBM_OK;
}

/* Pinned host memory for callers that want DMA-speed obm_lex_batch (the cgo shim keeps manifests in C memory). */
extern "C" void *obm_pinned_alloc(uint64_t bytes) { void *p = nullptr; return cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) == cudaSuccess ? p : nullptr; }
extern "C" void obm_pinned_free(void *p) { if (p) cudaFreeHost(p); }
