/*
 * obm_large.h -- documents larger than a tile (> obmt::MAXDOC bytes): chunk-parallel exact lexing.
 *
 * The reference lexer is sequential per document (internal/markers/lexer/lexer.go:43-49), but every line that
 * the lexer reaches in state `lex` is independent of what came before (SURVEY.md A.11).  A large document is cut
 * into chunks of LCHUNK bytes; chunk c starts at the first LINE START at or after c * LCHUNK and one thread lexes
 * line after line with the exact (Unicode) obm::Lexer in LINE mode -- the same composition tests/hostsim checks
 * as hs_lex_doc_by_lines -- until it reaches the start of chunk c + 1.  The assumption "my first line starts in
 * state lex" is CHECKED, not trusted: chunk c must stop exactly on chunk c + 1's start with no fatal error.  A
 * multi-line construct that crosses a chunk boundary overshoots it, the chain check fails and that document is
 * lexed sequentially instead (obm_lib.cu: k_large_resolve / k_large_fill).
 *
 * Host/device logic only; the kernels live in obm_lib.cu.  Compiled for the host by tests/hostsim.
 */
#ifndef OBM_LARGE_H
#define OBM_LARGE_H

#include "obm_core.h"

namespace obml {

constexpr uint32_t LCHUNK = 1024;
enum : uint32_t { CF_FATAL = 1, CF_OVERSHOOT = 2 };

OBM_HD uint32_t n_chunks(uint32_t len) { return len == 0 ? 1u : (uint32_t)(((uint64_t)len + LCHUNK - 1) / LCHUNK); }

/* start of chunk c, looked for inside the chunk only: the first line start (0, or the byte after a '\n') in
 * [c * LCHUNK, min((c + 1) * LCHUNK, n)], or n if the chunk holds none (resolve_chunk_starts then gives it the next
 * chunk's start).  Reading one chunk per call keeps the whole search linear in the document, however long its lines.
 * nl_skipped: newlines in [c * LCHUNK, start) */
OBM_HD uint32_t chunk_start(const uint8_t *doc, uint32_t n, uint32_t c, uint32_t *nl_skipped) {
    *nl_skipped = 0;
    if (c == 0) return 0;
    const uint64_t nominal = (uint64_t)c * LCHUNK;
    if (nominal >= n) return n;
    uint32_t p = (uint32_t)nominal;
    if (doc[p - 1] == '\n') return p;
    const uint32_t b = (n - p > LCHUNK) ? p + LCHUNK : n;
    while (p < b && doc[p] != '\n') p++;
    if (p >= b) return n;
    *nl_skipped = 1;
    return p + 1;
}

/* After chunk_start for every chunk of a document and line[c] = 1 + newlines before c * LCHUNK + nl_skipped: a chunk
 * c < nc - 1 with no line start of its own (start beyond its end, i.e. n) takes the start and the line of the next
 * chunk that has one.  That is the first line start at or after c * LCHUNK, so every chunk that lexes anything keeps
 * the start and line of a search that runs on past its end; the chunks that take over a start lex nothing. */
OBM_HD void resolve_chunk_starts(uint32_t *cs, uint32_t *line, uint32_t nc) {
    for (uint32_t k = nc - 1; k > 1; k--) { /* chunks nc - 2 .. 1, backwards */
        const uint32_t c = k - 1;
        if (cs[c] > (uint64_t)k * LCHUNK) { cs[c] = cs[k]; line[c] = line[k]; }
    }
}

/* newlines in [c * LCHUNK, min((c + 1) * LCHUNK, n)) */
OBM_HD uint32_t chunk_newlines(const uint8_t *doc, uint32_t n, uint32_t c) {
    const uint64_t a64 = (uint64_t)c * LCHUNK;
    if (a64 >= n) return 0;
    const uint32_t a = (uint32_t)a64, b = (n - a > LCHUNK) ? a + LCHUNK : n;
    uint32_t k = 0;
    for (uint32_t p = a; p < b; p++) k += doc[p] == '\n';
    return k;
}

/* lex / lexComment skipping for an all-ASCII document read from memory: the next position >= p whose byte is a
 * newline or one of # ' + / (a superset of what state.go:20-33,48 reacts to), 4 bytes per step on aligned words */
struct ChunkAccel {
    const uint8_t *d; uint32_t n;
    OBM_HD uint32_t next_interesting(uint32_t p) const {
        while (p < n) {
            const uint32_t mis = (uint32_t)((uintptr_t)(d + p) & 3u);
            const uint32_t w = *reinterpret_cast<const uint32_t *>(d + p - mis);
            const uint32_t hit = (zero4((w & 0xF3F3F3F3u) ^ 0x23232323u) | zero4(w ^ 0x0A0A0A0Au)) >> mis;
            if (hit) {
#if defined(__CUDA_ARCH__)
                const uint32_t q = p + (uint32_t)(__ffs((int)hit) - 1);
#else
                const uint32_t q = p + (uint32_t)__builtin_ctz(hit);
#endif
                return q < n ? q : n;
            }
            p += 4 - mis;
        }
        return n;
    }
    static OBM_HD uint32_t zero4(uint32_t t) { /* 4-bit mask of the zero bytes of t (bytes < 0x80) */
        const uint32_t ne = ((t + 0x7F7F7F7Fu) >> 7) & 0x01010101u;
        return ((ne ^ 0x01010101u) * 0x00204081u >> 21) & 0xFu;
    }
};

/* Lexes the lines of [start, stop) -- `line` is the 1-based number of the line at `start`, `stop` the start of
 * the next chunk (n for the last one).  Emits no EOF tuple.  Returns CF_* flags; *end is where the lexer stood. */
template <class Sink, bool ASCII = false>
OBM_HD uint32_t lex_chunk(const obm::Tables &T, const uint8_t *doc, uint32_t n, uint32_t start, uint32_t line, uint32_t stop, Sink &sink,
                          uint32_t *end) {
    /* ASCII: the whole document is < 0x80 (checked by the caller): the fast instantiation with word-wise skipping */
    uint32_t pos = start, ln = line;
    while (pos < stop) {
        int st; uint32_t np, nl;
        if constexpr (ASCII) {
            obm::Lexer<Sink, ChunkAccel, true> lx(T, doc, n, sink, pos, ln, pos, !(ln == 1 && pos == 0), ChunkAccel{doc, n});
            st = lx.template run<true>(); np = lx.p; nl = lx.line_p;
        } else {
            obm::Lexer<Sink> lx(T, doc, n, sink, pos, ln, pos, !(ln == 1 && pos == 0));
            st = lx.template run<true>(); np = lx.p; nl = lx.line_p;
        }
        if (st == obm::RUN_FATAL) { *end = np; return CF_FATAL; }
        if (st == obm::RUN_EOF) { pos = n; break; }
        pos = np; ln = nl;
    }
    *end = pos;
    return pos > stop ? (uint32_t)CF_OVERSHOOT : 0u;
}

/* any byte >= 0x80 in [c * LCHUNK, min((c + 1) * LCHUNK, n)) */
OBM_HD bool chunk_non_ascii(const uint8_t *doc, uint32_t n, uint32_t c) {
    const uint64_t a64 = (uint64_t)c * LCHUNK;
    if (a64 >= n) return false;
    const uint32_t a = (uint32_t)a64, b = (n - a > LCHUNK) ? a + LCHUNK : n;
    uint32_t acc = 0;
    for (uint32_t p = a; p < b; p++) acc |= doc[p];
    return (acc & 0x80u) != 0;
}

} /* namespace obml */
#endif
