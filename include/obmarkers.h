/*
 * obmarkers.h -- C ABI of libobmarkers.so, the H100 (sm_90a) marker scanner.
 *
 * Drop-in boundary for the marker-scanning hot path of vmware-tanzu-labs/operator-builder
 * (reference @ 2827f233; file:line citations are relative to the reference tree).
 *
 * The reference has no FFI at this seam; the seam is three exported Go methods consumed only by
 * internal/markers/parser:
 *     func NewLexer(r io.Reader) *Lexer          internal/markers/lexer/lexer.go:27
 *     func (l *Lexer) Run()                      internal/markers/lexer/lexer.go:43
 *     func (l *Lexer) NextLexeme() Lexeme        internal/markers/lexer/lexer.go:51
 *     type Lexeme struct{Type; Value; Pos}       internal/markers/lexer/lexeme.go:32-36
 * A cgo shim (operator-builder_b200/go/lexer_gpu.go, INTEGRATION.md) keeps that surface and feeds it
 * from the entry points below: one obm_lex_batch() per `create api` replaces one lexer goroutine
 * per YAML node (internal/markers/inspect/yaml.go:94), and obm_stream_* replays a document's
 * tuples as the exact Lexeme sequence the Go lexer would have sent on its channel.
 *
 * All entry points use plain pointers and sizes.  The callee keeps no pointer after return (cgo
 * rule).  Lexical errors/warnings are IN-BAND tuples (the reference sends them in-band as
 * LexemeError / LexemeWarning, lexer/error.go:15-45); infrastructure failures (CUDA, capacity,
 * arguments) are negative return codes plus obm_last_error().
 *
 * There is no CPU fallback: every lexing entry point fails with OBM_E_NO_DEVICE when no CUDA
 * device is usable.  obm_stream_* / obm_parse_* are host-side consumers of tuples the GPU produced.
 */
#ifndef OBMARKERS_H
#define OBMARKERS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OBM_ABI_VERSION 1

/* ---------------------------------------------------------------------------------------------
 * Tuple stream.  One 64-bit little-endian word per tuple:
 *     bits  0..31  off   byte offset inside the document
 *     bits 32..58  len   byte length (27 bits)
 *     bits 59..63  kind
 * Kinds 0..20 are the reference's LexemeType values (lexer/lexeme.go:8-30).  Kinds 21..29 are
 * pseudo-tuples the host decoder folds away so that the decoded stream is byte-identical to the
 * reference's (Type, Value, Pos) sequence, including its implementation artefacts:
 *   PART    text that sits in the reference lexer's `buffer` without having been emitted; it is
 *           prepended to the Value of the next real lexeme (emit.go:8-17 clears buffer only on emit)
 *   FLUSH   the reference called flush() (discard.go:68-71; state.go:81,128)
 *   DRIFT   the second backup() of state.go:79/126 shortened the column by one (position.go:44-45)
 *   LINE    position basis: off = byte offset of column 1, len = line number (low 27 bits);
 *           emitted before the first located tuple that is not on the previously announced line
 *   LINEHI  high bits (>> 27) of the next LINE's line number (documents with > 134M lines)
 *   WARN_ / ERR_  in-band warnings / fatal errors; the decoder formats the reference's exact text
 * Kinds 0 (Error) and 19 (Warning) never appear raw; 14..17 are never emitted by the reference.
 * ------------------------------------------------------------------------------------------- */
typedef uint64_t obm_tuple;

enum obm_kind {
    OBM_K_ERROR = 0, OBM_K_COMMENT = 1, OBM_K_MARKER_START = 2, OBM_K_SCOPE = 3, OBM_K_SEPARATOR = 4,
    OBM_K_ARG = 5, OBM_K_ARG_ASSIGNMENT = 6, OBM_K_ARG_DELIMITER = 7, OBM_K_STRING_LITERAL = 8,
    OBM_K_FLOAT_LITERAL = 9, OBM_K_INTEGER_LITERAL = 10, OBM_K_SYNTHETIC_BOOL = 11, OBM_K_BOOL_LITERAL = 12,
    OBM_K_QUOTE = 13, OBM_K_MARKER_END = 18, OBM_K_WARNING = 19, OBM_K_EOF = 20,
    OBM_K_PART = 21, OBM_K_FLUSH = 22, OBM_K_DRIFT = 23, OBM_K_LINE = 24, OBM_K_LINEHI = 25,
    OBM_K_WARN_NOSCOPE = 26,   /* "marker without scope found"  state.go:95,105 ; off = position */
    OBM_K_WARN_INVALID = 27,   /* "invalid marker found"        state.go:114    ; off = position */
    OBM_K_ERR_MALFORMED = 28,  /* "malformed argument: %s"      state.go:152,173,315 ; off = position */
    OBM_K_ERR_UNMATCHED = 29,  /* "unmatched string delimiter"  state.go:193,199,209 ; off = position */
    OBM_K_ERR_FLOAT = 30,      /* "invalid float literal"       state.go:259 ; off,len = the literal */
    OBM_K_ERR_INT = 31         /* "invalid integer literal"     state.go:270 ; off,len = the literal */
};

#define OBM_LEN_BITS 27
#define OBM_MAX_LEN ((1u << OBM_LEN_BITS) - 1u)
#define OBM_TUPLE(kind, off, len) (((uint64_t)(kind) << 59) | ((uint64_t)(len) << 32) | (uint64_t)(uint32_t)(off))
#define OBM_TUPLE_KIND(t) ((unsigned)((t) >> 59))
#define OBM_TUPLE_LEN(t) ((uint32_t)(((t) >> 32) & OBM_MAX_LEN))
#define OBM_TUPLE_OFF(t) ((uint32_t)((t) & 0xFFFFFFFFu))

/* A document may be at most 2^31 - 2 bytes: offsets are 32-bit inside a document and the per-document tuple counts are
 * 32-bit too (the grammar emits up to 1.5 tuples per byte: ",c" is Arg + SyntheticBool + ArgDelimiter). */
#define OBM_MAX_DOC_BYTES 0x7FFFFFFEull

/* return codes */
enum obm_status {
    OBM_OK = 0,
    OBM_E_NO_DEVICE = -1,   /* no CUDA device / driver: there is no CPU fallback */
    OBM_E_CUDA = -2,        /* a CUDA call failed; see obm_last_error */
    OBM_E_CAPACITY = -3,    /* `out_cap` too small; *out_count holds the required tuple count */
    OBM_E_ARG = -4,         /* bad argument (null pointer, non-monotonic doc_off, oversize document) */
    OBM_E_NOMEM = -5
};

typedef struct obm_handle obm_handle;
typedef struct obm_registry obm_registry; /* marker.Registry stand-in, below */

/* Counters filled by a scan (all per call). */
typedef struct obm_stats {
    uint64_t n_tuples;        /* tuples written (incl. pseudo-tuples) */
    uint64_t n_markers;       /* MarkerStart lexemes  */
    uint64_t n_lexemes;       /* real lexemes a reference lexer would have sent (incl. EOF/warnings/errors) */
    uint64_t n_docs_exact;    /* documents that took the exact (sequential) device path */
    uint64_t n_docs_fatal;    /* documents that ended in a fatal lexical error */
    uint64_t bytes;           /* input bytes scanned */
    float    ms_kernels;      /* device time of the scan kernels (CUDA events), host-buffer calls also: */
    float    ms_total;        /* H2D + kernels + D2H as seen by CUDA events on the handle's stream */
} obm_stats;

/* --- lifetime ------------------------------------------------------------------------------ */
int obm_abi_version(void);
/* Creates a scanner bound to CUDA device `device_ordinal` with its own stream. */
int obm_create(int device_ordinal, obm_handle **out);
void obm_destroy(obm_handle *h);
/* Message of the last failure on this handle (or a static message when h is NULL). */
const char *obm_last_error(const obm_handle *h);

/* --- the hot path -------------------------------------------------------------------------- */
/*
 * Lex a packed batch of documents held in HOST memory (replaces, for every document d,
 * lexer.NewLexer(bytes.NewBuffer(bytes[doc_off[d]:doc_off[d+1]])) + Run + drain, lexer.go:27-53).
 *   bytes        packed documents, back to back
 *   doc_off      ndocs+1 ascending byte offsets into `bytes`
 *   out          receives tuples; document d's tuples are out[doc_tuple_off[d] .. doc_tuple_off[d+1])
 *   out_cap      capacity of `out` in tuples.  If too small: returns OBM_E_CAPACITY with the needed
 *                count in *out_count and doc_tuple_off filled; the contents of `out` are then unspecified (the
 *                chunked path may already have copied the tuples of earlier chunks).
 *                Pass out = NULL, out_cap = 0 to size a buffer.
 *   stats        optional
 */
int obm_lex_batch(obm_handle *h, const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs,
                  obm_tuple *out, uint64_t out_cap, uint64_t *out_count, uint64_t *doc_tuple_off,
                  obm_stats *stats);

/*
 * Same scan on DEVICE-resident buffers (benchmarking / pipelines that keep manifests in HBM).
 * All pointers are device pointers on the handle's device; `stream` is a cudaStream_t used exactly as
 * given (NULL = CUDA's default stream).  Asynchronous: returns after enqueueing.  d_doc_tuple_off[ndocs] holds the
 * total tuple count; if it exceeds out_cap the kernels write nothing past out_cap and set
 * d_status[0] = 1 (d_status is a device uint32[4]: {overflow, n_docs_exact, n_docs_fatal, scratch_overflow}).
 * scratch_overflow != 0 means the pipeline's internal work-record buffers were too small: the output is invalid,
 * rerun with obm_set_mode(h, 1).  The capacities behind obm_scratch_bytes are structural bounds, so this is a
 * defensive check, not an expected outcome (obm_lex_batch reruns by itself).
 * d_bytes must be readable from the 16-byte boundary at or before it up to the next 16-byte boundary past
 * d_bytes + total_bytes (any cudaMalloc'd buffer is): TMA, cp.async and aligned vector loads round to 16 bytes.
 * d_counts (device uint64[2], may be NULL) receives {n_markers, n_lexemes}.
 */
int obm_lex_batch_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                         uint64_t total_bytes, void *d_out, uint64_t out_cap, void *d_doc_tuple_off,
                         void *d_status, void *d_counts, void *stream);

/* Bytes of device scratch obm_lex_batch_device needs for `ndocs`/`total_bytes` (allocated lazily,
 * grown on demand and kept by the handle). */
uint64_t obm_scratch_bytes(uint32_t ndocs, uint64_t total_bytes);

/* Deterministic synthetic corpus generated ON DEVICE (BASELINE.md config C2/C3/C4 generator; the
 * same generator exists on the host: obm_generate_corpus_host below, oracle/corpus_gen.cpp for the reference arm).
 * Writes ndocs documents of exactly doc_bytes bytes starting at global document index first_doc.
 * flavour: 0 = standalone markers, 1 = collection markers. */
int obm_generate_corpus_device(obm_handle *h, void *d_bytes, void *d_doc_off, uint32_t ndocs,
                               uint32_t doc_bytes, uint64_t first_doc, int flavour, void *stream);

/* Host copy of the same generator (test / bench utility; performs no lexing). */
int obm_generate_corpus_host(uint8_t *bytes, uint64_t *doc_off, uint32_t ndocs, uint32_t doc_bytes,
                             uint64_t first_doc, int flavour);

/* Scanning strategy: 0 = fused warp kernel (default; csrc/obm_warp.h), 1 = exact path for every document,
 * 2 = round 1's fused tile kernel, 3 = round 1's two-stage pipeline (keeps valid UTF-8 documents line-parallel).
 * All produce the identical tuple stream.  Returns the old mode. */
int obm_set_mode(obm_handle *h, int mode);

/* obm_lex_batch pipelines host batches of at least two chunks: H2D of chunk k+1, the scan of chunk k and D2H of
 * chunk k-1 overlap on three streams (pass pinned buffers, obm_pinned_alloc, for the copies to be asynchronous).
 * Default chunk: 64 MiB (env OBM_CHUNK_MB).  Returns the previous value. */
uint64_t obm_set_chunk_bytes(obm_handle *h, uint64_t bytes);

/* Number of this library's kernels launched by the last scan call on this handle. */
uint32_t obm_launches_last_call(const obm_handle *h);

/* Page-locked host memory so that obm_lex_batch's copies run at DMA speed (the cgo shim keeps
 * manifest bytes in C memory anyway). */
void *obm_pinned_alloc(uint64_t bytes);
void obm_pinned_free(void *p);

/* --- the data formats either side of the scan (SURVEY.md 8(f) ranks 2 and 4), device resident ------------ */
/*
 * Manifest.LoadContent's collection rewrite (internal/workload/v1/manifests/manifest.go:89-95):
 *     ReplaceAll(content, "+operator-builder:collection:field", "+operator-builder:field")
 *     ReplaceAll(content, "collectionField", "field")
 * applied to every document of a packed batch in HBM.  Writes the rewritten batch (never longer than the
 * input) and its ndocs+1 offsets; with d_out_bytes == NULL only the offsets are produced.  One pass over the batch
 * (csrc/obm_rewrite.cuh) when d_bytes and d_out_bytes are 16-byte aligned, two passes over the documents otherwise.
 * Nothing is written past out_cap; OBM_E_CAPACITY reports an output that did not fit.  Synchronises the stream.
 * (Test switch: OBM_REWRITE_TWO_PASS=1 in the environment forces the two-pass path.)
 */
int obm_rewrite_collection_markers_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                                          void *d_out_bytes, uint64_t out_cap, void *d_out_doc_off, void *stream);
/*
 * The collection rewrite above and the scan of its result, for device-resident collection batches: one call that is
 * defined as these two calls, in every mode (obm_set_mode applies to the scan)
 *     obm_rewrite_collection_markers_device(h, d_bytes, d_doc_off, ndocs, d_out_bytes, out_bytes_cap, d_out_doc_off, stream)
 *     obm_lex_batch_device(h, d_out_bytes, d_out_doc_off, ndocs, <rewritten total>, d_out, out_cap, d_doc_tuple_off,
 *                          d_status, d_counts, stream)
 * i.e. the rewritten bytes and d_out_doc_off[ndocs+1], the tuple stream of the REWRITTEN documents (offsets relative to
 * them), d_doc_tuple_off, status and counts with obm_lex_batch_device's semantics.
 * d_bytes: as for obm_lex_batch_device.  d_out_bytes: 16-byte aligned, not overlapping d_bytes, out_bytes_cap >=
 * total_bytes (the rewrite never lengthens the text, so the bytes cannot overflow); OBM_E_ARG otherwise.  Nothing is
 * written at or past d_out_doc_off[ndocs] in d_out_bytes.  Synchronises the stream: the rewritten total, which sizes
 * the scan, is read back between the two calls.
 */
int obm_lex_collection_batch_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, uint64_t total_bytes,
                                    void *d_out_bytes, uint64_t out_bytes_cap, void *d_out_doc_off,
                                    void *d_out, uint64_t out_cap, void *d_doc_tuple_off, void *d_status, void *d_counts, void *stream);
/*
 * Manifest.ExtractManifests (manifests/manifest.go:57-80): split every document on lines that equal "---" after
 * trimming trailing spaces.  One 16-byte record {u32 doc, u32 a, u32 b, u32 0} per extracted manifest, whose text
 * is "\n" + content[a:b) exactly as the reference rebuilds it; d_doc_rec_off[ndocs+1] = per-document offsets.
 */
int obm_split_docs_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, void *d_records, uint64_t cap,
                          void *d_doc_rec_off, void *stream);

/* --- multi-GPU: manifests shard by file (lexer.go:27-40: one lexer per input), one rank per GPU ------------------
 * The one exchange step of the path is an NCCL all-gather over NVLink of the shard's compact index of registered
 * markers (16 bytes per marker, ~3 % of the input) -- the full tuple stream (~35 %) stays resident on its owner.  NCCL is loaded at run time (libnccl.so.2); the caller moves the 128-byte unique id from rank 0 to the other
 * ranks by whatever channel it has (the Go host: its own RPC; bench.py: torch.distributed).                         */
typedef struct obm_comm obm_comm;
#define OBM_COMM_ID_BYTES 128
int obm_comm_unique_id(uint8_t *id /* OBM_COMM_ID_BYTES */);
int obm_comm_create(obm_handle *h, const uint8_t *id, int rank, int nranks, obm_comm **out);
void obm_comm_destroy(obm_comm *c);
/*
 * One sharded step on this rank's device-resident shard (documents first_doc .. first_doc + ndocs of the global batch):
 * scan (obm_lex_batch_device), the compact index of the registered markers (obm_marker_index_flat_device; records carry
 * global document ids), then ONE ncclAllGather of the 16-byte index records.  d_index_all receives nranks slots of
 * *stride records each (stride = the largest per-rank count, chosen inside: an 8-byte count all-gather + host read);
 * rank_records[r] = valid records of slot r.  Returns OBM_E_CAPACITY (with *stride set) when index_cap < this rank's
 * count or index_all_cap < nranks * stride.  The shard's tuples and offsets stay in the caller's buffers (d_out, ...):
 * the index says which rank and which tuple to ask for.  The collective is enqueued on `stream`.
 */
int obm_lex_batch_sharded_device(obm_comm *c, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                                 uint64_t total_bytes, uint32_t first_doc, void *d_out, uint64_t out_cap, void *d_doc_tuple_off, void *d_status,
                                 void *d_counts, void *d_index, uint64_t index_cap, void *d_index_all, uint64_t index_all_cap,
                                 uint64_t *rank_records /* host u64[nranks] */, uint64_t *stride, void *stream);

/* --- host-side consumers of the tuple stream (no GPU needed; no lexing happens here) ------- */
/*
 * Replays one document's tuples as the reference's Lexeme sequence.  Mirrors
 * NewLexer/Run/NextLexeme: after the last lexeme (EOF, or a fatal Error) obm_stream_next returns 0
 * and yields the zero Lexeme {Type: 0, Value: ""} like a closed Go channel (lexer.go:47,51-53).
 */
typedef struct obm_stream obm_stream;
typedef struct obm_lexeme {
    int32_t type;          /* reference LexemeType 0..20 */
    const uint8_t *value;  /* valid until the next call on this stream */
    uint64_t value_len;
    int64_t line, column;  /* Pos; {0,0} for synthetic lexemes (emit.go:24-33) */
} obm_lexeme;
obm_stream *obm_stream_new(const uint8_t *doc, uint64_t doc_len, const obm_tuple *tuples, uint64_t ntuples);
int obm_stream_next(obm_stream *s, obm_lexeme *out); /* 1 = lexeme produced, 0 = stream closed */
void obm_stream_free(obm_stream *s);
/*
 * Decodes a whole document into a flat buffer of records
 *     [u8 type][u32 line][u32 col][u32 vlen][value bytes] ...
 * (*out is malloc'd; release with obm_free).  Returns the number of lexemes or a negative status.
 */
int64_t obm_decode_doc(const uint8_t *doc, uint64_t doc_len, const obm_tuple *tuples, uint64_t ntuples,
                       uint8_t **out, uint64_t *out_len);
void obm_free(void *p);

/*
 * The lexer's only consumer on the same tuple stream (SURVEY.md 8(f) rank 1): mirrors internal/markers/parser
 * (state.go:13-175, definition.go:13-21, emit.go:8-24, error.go:8-22) over obm_stream_*.  A registry lists the
 * marker names (with their leading '+', e.g. "+operator-builder:field") and the argument names each accepts
 * (marker/marker.go LookupArgument).  obm_parse_doc returns the number of Results and a malloc'd record
 * buffer (format: csrc/obm_parse.cpp).
 * A definition added with names only (obm_registry_add, obm_registry_operator_builder) accepts every value: each
 * SetArgument succeeds and emit() always succeeds.  A definition added by obm_registry_define carries the Go types of
 * marker.Define(name, T{}) and gets the reference's SetArgument (marker/argument.go:91-127: wrong type, the FieldType
 * unmarshal error, the int -> string reflect.Set panic) and InflateObject (marker/marker.go:65-95: missing required
 * arguments).  Parity unpinned: the reference has no parser tests; only the FieldType names are pinned
 * (field_types_internal_test.go).  Go lists missing arguments in map order; here they are in definition order.
 */
obm_registry *obm_registry_new(void);
obm_registry *obm_registry_operator_builder(void); /* field / collection:field / resource markers, names only */
int obm_registry_add(obm_registry *r, const char *marker_name, const char *const *arg_names, uint32_t nargs);
/* internal/workload/v1/markers/markers.go:20-25 (MarkerType) and :92-113 (the definition each adds) */
enum { OBM_FIELD_MARKER = 0, OBM_COLLECTION_MARKER = 1, OBM_RESOURCE_MARKER = 2 };
/* Adds the typed definition of one marker type; defining a name again replaces it (Registry.Add, marker/registry.go:20-22).
 * Build InspectForYAML's subsets this way, e.g. resource only (child_resource.go:71).  OBM_E_ARG for another type. */
int obm_registry_define(obm_registry *r, int marker_type);
void obm_registry_free(obm_registry *r);
/*
 * Device side of the same row: a compact index of the REGISTERED markers in a tuple stream that is still in
 * HBM -- one 16-byte record {u32 doc, u32 tuple index in the document, u32 offset of '+', u16 registry id,
 * u16 scope count} per marker whose name parser/definition.go:13-21 would find in the registry (at most 8
 * names, 512 bytes: more is OBM_E_ARG).  d_doc_rec_off[ndocs+1] receives the per-document record offsets (last =
 * total); records beyond `cap` are not written -- compare the total with cap (the same holds for obm_split_docs_device).
 * With d_records == NULL only the offsets are computed.  These next-row entry points use the handle's scratch: enqueue
 * them on the stream the handle's scans run on (one stream per handle).  This index (~3 % of the input), not the tuple stream
 * (~35 %), is what ranks exchange over NVLink.
 */
int obm_marker_index_device(obm_handle *h, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs,
                            const void *d_tuples, const void *d_doc_tuple_off, void *d_records, uint64_t cap,
                            void *d_doc_rec_off, void *stream);
/* The same records (document order, doc_base added to the document ids) from ONE flat pass over the tuple stream (2,048-tuple
 * tiles, the rare MarkerStart candidates examined a thread each, tile totals through a look-back) instead of a warp per
 * document: ~6x faster; no per-document offsets.  ntuples_bound: an upper bound of the stream's
 * length known on the host (the capacity of d_tuples does); *d_total (device u64) = number of records. */
int obm_marker_index_flat_device(obm_handle *h, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, uint32_t doc_base,
                                 const void *d_tuples, const void *d_doc_tuple_off, uint64_t ntuples_bound, void *d_records, uint64_t cap,
                                 void *d_total, void *stream);
/*
 * The same consumer ON THE DEVICE (csrc/obm_parse_dev.h): one thread per document walks the resident tuple stream as
 * parser/state.go:13-175 walks lexemes -- registry lookup (definition.go:13-21), known-argument filter
 * (state.go:79-93), value typing (ParseBool / Atoi class / ParseFloat(., 32) range, state.go:95-153), MarkerText as a
 * span of the document, error results (error.go:8-22) -- and writes compact records:
 *   obm_result (32 B)  one per Result, document order; obm_arg (16 B) one per accepted argument
 * Documents whose stream holds pseudo-tuples the walk does not model (stale-buffer PART / FLUSH, DRIFT, LINEHI, in-band
 * warnings, lexer errors) get ONE record with OBM_R_HOST: run obm_parse_doc on that document (exact for everything).
 * d_doc_res_off[ndocs+1]: per-document result offsets; d_totals: device u64[2] = {results, args}.  With d_results ==
 * NULL only the offsets / totals are computed.  doc_base is added to every record's doc (global ids of a shard).
 */
typedef struct obm_result {
    uint32_t doc;        /* document index + doc_base */
    uint32_t tuple;      /* index, inside the document, of the marker's MarkerStart tuple (error results: parser.current) */
    uint32_t text_off;   /* MarkerText = doc[text_off, text_off + text_len) (+ "\n" when OBM_R_NL) */
    uint32_t text_len;
    uint16_t reg_id;     /* registry entry; 0xFFFF on OBM_R_HOST records */
    uint16_t nargs;      /* error results: 1 = {name_off: line, val_off/val_len: the offending literal}; OBM_R_ERR_MISSING: 0 */
    uint32_t arg_base;   /* index of the first obm_arg of this result in the batch's argument array */
    uint32_t flags;      /* OBM_R_* */
    uint32_t aux;        /* error results: column of parser.current; OBM_R_HOST: the first unmodelled tuple kind;
                            OBM_R_ERR_MISSING: bit j = the definition's argument j is required and was never set */
} obm_result;
typedef struct obm_arg {
    uint32_t name_off;   /* argument name = doc[name_off, name_off + name_len) */
    uint32_t val_off;    /* value = doc[val_off, val_off + val_len); OBM_A_SYNTHETIC_TRUE: the value is "true" */
    uint32_t val_len;
    uint16_t name_len;   /* OBM_R_ERR_SETARG / OBM_R_PANIC: the argument's index in its definition (name_off: line) */
    uint8_t kind;        /* 0 bool, 1 int, 2 float, 3 string */
    uint8_t flags;
} obm_arg;
/* Typed definitions only (obm_registry_define):
 *   OBM_R_ERR_SETARG   SetArgument failed: wrong type or FieldType unmarshal error (the formatter derives which from the
 *                      argument's type and the value); ends the document's parse like the strconv errors
 *   OBM_R_ERR_MISSING  InflateObject: required arguments never set (mask in aux); position {line:0 column:0}, MarkerText
 *                      ends in the synthetic "\n" (OBM_R_NL); ends the document's parse
 *   OBM_R_PANIC        SetArgument would panic in reflect.Set (an int for a string argument).  Not a Result in the
 *                      reference: its process aborts.  Treat it as fatal for the whole run.
 *   OBM_A_SUPERSEDED   an argument a later one of the same name overwrote (marker.go:59): the arguments of an OK result
 *                      without it are exactly the fields InflateObject sets */
enum { OBM_R_OK = 1, OBM_R_NL = 2, OBM_R_ERR_PARSEBOOL = 4, OBM_R_ERR_FLOAT32 = 8, OBM_R_HOST = 16, OBM_R_ERR_SETARG = 32,
       OBM_R_ERR_MISSING = 64, OBM_R_PANIC = 128 };
enum { OBM_A_SYNTHETIC_TRUE = 1, OBM_A_SUPERSEDED = 2 };
/*
 * Per-document 64-bit hash of the DECODED lexeme stream, computed on the device from the resident tuples: FNV-1a over
 * the records [u8 type][u32 line][u32 col][u32 vlen][value] that obm_decode_doc serialises (and that the reference
 * lexer would send: Type, Pos, Value).  Lets a full-size batch (4 GiB, 10 GiB) be checked document by document against a
 * CPU run without moving the tuples.  Documents the device walk does not model (pseudo-tuples other than LINE, bytes
 * >= 0x80 inside a value) get hash 0 and are counted in *d_n_host (device u32): hash those from obm_decode_doc.
 */
int obm_hash_batch_device(obm_handle *h, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, const void *d_tuples,
                          const void *d_doc_tuple_off, void *d_hashes /* u64[ndocs] */, void *d_n_host, void *stream);
int obm_parse_batch_device(obm_handle *h, const obm_registry *reg, const void *d_bytes, const void *d_doc_off, uint32_t ndocs, uint32_t doc_base,
                           const void *d_tuples, const void *d_doc_tuple_off, void *d_results, uint64_t res_cap, void *d_args, uint64_t arg_cap,
                           void *d_doc_res_off, void *d_totals, void *stream);
/* Records of ONE document -> the byte format of obm_parse_doc (so both can be compared / consumed alike); documents
 * flagged OBM_R_HOST are parsed from `tuples` by obm_parse_doc itself.  Returns the number of Results. */
int64_t obm_results_format_doc(const obm_registry *reg, const uint8_t *doc, uint64_t doc_len, const obm_tuple *tuples, uint64_t ntuples,
                               const obm_result *results, uint64_t nresults, const obm_arg *args_base /* the batch's array */,
                               uint8_t **out, uint64_t *out_len);
int64_t obm_parse_doc(const obm_registry *reg, const uint8_t *doc, uint64_t doc_len, const obm_tuple *tuples, uint64_t ntuples,
                      uint8_t **out, uint64_t *out_len);
/*
 * Parse a packed batch held in HOST memory on the device: H2D, the scan, obm_parse_batch_device and the D2H of the
 * records only -- the tuple stream stays on the device except for the documents the host must parse itself.
 *   results / args   exactly what obm_parse_batch_device writes for the same batch with doc_base = 0: `doc` is the
 *                    document index in this batch, arg_base indexes `args` as a whole, spans are document-relative.
 *                    Document d's Results are results[doc_res_off[d] .. doc_res_off[d+1]).
 *   host_tuples      for every document whose one record is OBM_R_HOST, its whole tuple stream (as obm_lex_batch returns
 *                    it) in host_tuples[doc_host_off[d] .. doc_host_off[d+1]); that range is empty for every other
 *                    document.  So for every d,
 *                        obm_results_format_doc(reg, doc_d, len_d, host_tuples + doc_host_off[d], doc_host_off[d+1] - doc_host_off[d],
 *                                               results + doc_res_off[d], doc_res_off[d+1] - doc_res_off[d], args, ...)
 *                    gives obm_parse_doc's bytes for that document.
 *   totals           [3]: results, args, fallback tuples.
 * Capacities as in obm_lex_batch: NULL or 0 capacities size the buffers; when any total exceeds its capacity the call
 * returns OBM_E_CAPACITY with totals, doc_res_off and doc_host_off (ndocs+1 each) filled, and writes nothing past any
 * capacity (the arrays' contents are then unspecified).  The registry is limited as for the device parser (8 markers, 64
 * arguments, 1024 bytes of names), else OBM_E_ARG; doc_off is checked as by obm_lex_batch; ndocs = 0 is valid.
 * obm_set_mode applies to the scan (a scratch overflow redoes the chunk in mode 1, as obm_lex_batch does), and batches of
 * at least two chunks (obm_set_chunk_bytes) are pipelined over obm_lex_batch's three streams.  stats: the scan counters,
 * bytes, ms_kernels = scan + parse + gather (summed over chunks), ms_total.  obm_launches_last_call counts every kernel of
 * the call, over all its chunks.
 */
int obm_parse_batch(obm_handle *h, const obm_registry *reg, const uint8_t *bytes, const uint64_t *doc_off, uint32_t ndocs,
                    obm_result *results, uint64_t res_cap, obm_arg *args, uint64_t arg_cap, uint64_t *doc_res_off /* ndocs+1 */,
                    obm_tuple *host_tuples, uint64_t host_cap, uint64_t *doc_host_off /* ndocs+1 */,
                    uint64_t *totals /* [3]: results, args, host tuples */, obm_stats *stats);

#ifdef __cplusplus
}
#endif
#endif /* OBMARKERS_H */
