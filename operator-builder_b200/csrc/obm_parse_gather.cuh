/*
 * obm_parse_gather.cuh -- the device side of obm_parse_batch around k_parse_docs (obm_parse_dev.h): what a host caller
 * needs next to the Result records, so that only records, offsets and fallback tuples cross PCIe.
 *   k_fallback_counts  per document: its tuple count when its one record is OBM_R_HOST (the host parses it from
 *                      its tuples), else 0; scanned into the fallback offsets with k_scan_tiles / k_scan_sums / k_scan_add
 *   k_fallback_gather  copies those documents' tuples, back to back, a warp per document
 *   k_rebase_records   turns a chunk's records and offsets into the batch's: adds the global bases of the chunk
 */
#ifndef OBM_PARSE_GATHER_CUH
#define OBM_PARSE_GATHER_CUH

namespace obmg {

constexpr uint32_t THREADS = 256;

__global__ void __launch_bounds__(THREADS)
k_fallback_counts(const obm_result *__restrict__ res, const uint64_t *__restrict__ res_off, const uint64_t *__restrict__ tuple_off,
                  uint32_t ndocs, uint32_t *__restrict__ counts) {
    for (uint32_t d = blockIdx.x * THREADS + threadIdx.x; d < ndocs; d += gridDim.x * THREADS) {
        const uint64_t r0 = res_off[d];
        const bool host = res_off[d + 1] > r0 && (res[r0].flags & OBM_R_HOST);
        counts[d] = host ? (uint32_t)(tuple_off[d + 1] - tuple_off[d]) : 0u;
    }
}

/* A warp per document rather than a flat pass over the output: fallback documents are few and each is one contiguous
 * run on both sides, so a warp copies it with coalesced 256-byte accesses, and every other document costs the warp one
 * pair of offset loads.  A flat pass would have to find each output tuple's document by a search over the offsets. */
__global__ void __launch_bounds__(THREADS)
k_fallback_gather(const obm_tuple *__restrict__ tuples, const uint64_t *__restrict__ tuple_off, const uint64_t *__restrict__ host_off,
                  uint32_t ndocs, obm_tuple *__restrict__ out) {
    const uint32_t lane = threadIdx.x & 31, nwarps = gridDim.x * (THREADS / 32);
    for (uint32_t d = blockIdx.x * (THREADS / 32) + (threadIdx.x >> 5); d < ndocs; d += nwarps) {
        const uint64_t h0 = host_off[d], n = host_off[d + 1] - h0;
        if (n == 0) continue;
        const obm_tuple *src = tuples + tuple_off[d];
        for (uint64_t k = lane; k < n; k += 32) out[h0 + k] = src[k];
    }
}

/* arg_base of every record but OBM_R_HOST ones (which carry 0 and index nothing) += arg_base_add (32-bit, as the
 * field is: the sum wraps exactly like the single-shot value does); res_off[0..ndocs) += res_base, host_off[0..ndocs)
 * += host_base.  Documents already carry global ids: the chunk was parsed with doc_base = its first document. */
__global__ void __launch_bounds__(THREADS)
k_rebase_records(obm_result *__restrict__ res, uint64_t nres, uint32_t arg_base_add, uint64_t *__restrict__ res_off,
                 uint64_t res_base, uint64_t *__restrict__ host_off, uint64_t host_base, uint32_t ndocs) {
    const uint64_t n = nres > ndocs ? nres : ndocs;
    for (uint64_t i = (uint64_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += (uint64_t)gridDim.x * THREADS) {
        if (i < nres && !(res[i].flags & OBM_R_HOST)) res[i].arg_base += arg_base_add;
        if (i < ndocs) { res_off[i] += res_base; host_off[i] += host_base; }
    }
}

} /* namespace obmg */
#endif
