/*
 * vlscan.h -- C ABI of the H100-native LogsQL block-scan / filter engine (libvlscan.so).
 *
 * Drop-in boundary for lib/logstorage's query hot path.  The reference has no FFI seam; it is cut at the body of the
 * search-worker loop over one blockSearchWorkBatch (lib/logstorage/storage_search.go:1044-1062): a batch of
 * independent blocks sharing one searchOptions.filter goes in, one row bitmap per block comes out, and everything
 * after it (blockResult.mustInit, initColumns, writeBlock) keeps working unchanged.  All file:line citations are
 * relative to the VictoriaLogs reference tree.  INTEGRATION.md shows the cgo binding a maintainer would add.
 *
 * Conventions (mirroring the reference's only FFI precedent, vendor/github.com/valyala/gozstd/gozstd.go:14-38):
 *   - plain pointers + sizes, no C++ / torch types; the library never retains caller pointers past return;
 *   - int return: 0 OK, <0 malformed input (the Go side turns it into logger.Panicf("FATAL: ...") like
 *     block_search.go:264,318,423,466), >0 CUDA error; text via vlscan_last_error();
 *   - re-entrant across distinct vlscan_ctx; one ctx <-> one calling thread (= one search worker goroutine).
 *   - there is NO CPU fallback: every entry point that computes fails with an error when no CUDA device is usable.
 */
#ifndef VLSCAN_H
#define VLSCAN_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct vlscan_ctx vlscan_ctx;         /* per search-worker state: device, stream, staging buffers          */
typedef struct vlscan_program vlscan_program; /* compiled filter tree (replaces so.filter, storage_search.go:1035)  */
typedef struct vlscan_batch vlscan_batch;     /* a batch of blocks resident in HBM                                  */

/* valueType, lib/logstorage/values_encoder.go:20-60 */
enum {
    VLSCAN_VT_STRING = 1, VLSCAN_VT_DICT = 2, VLSCAN_VT_UINT8 = 3, VLSCAN_VT_UINT16 = 4, VLSCAN_VT_UINT32 = 5,
    VLSCAN_VT_UINT64 = 6, VLSCAN_VT_FLOAT64 = 7, VLSCAN_VT_IPV4 = 8, VLSCAN_VT_ISO8601 = 9, VLSCAN_VT_INT64 = 10
};

/* column kinds: what blockSearch.getConstColumnValue / getColumnHeader would find (block_search.go:232-324).
 * A field that is absent from the block is simply not listed. */
enum { VLSCAN_COL_CONST = 1, VLSCAN_COL_VALUES = 2 };

/* stage of the values payload handed over */
enum {
    VLSCAN_STAGE_ONDISK = 0,  /* `values` = the bytes at [valuesOffset, +valuesSize) of the values file:
                                 bytesBlock(uintBlock lens) ++ bytesBlock(data), plain or ZSTD
                                 (lib/logstorage/encoding.go:16-50,343-426); the bytes go to HBM as they are and the
                                 ZSTD frames are decoded there (where the reference calls cgo libzstd per block)    */
    VLSCAN_STAGE_DECODED = 1  /* `lens_items` / `data` = what unmarshalBytesBlock yields for the two sub-blocks
                                 (encoding.go:372-426): the uintBlock items incl. their type byte, and the data     */
};

/* One column of one block: the fields of columnHeader the scan needs (lib/logstorage/block_header.go:584-615) plus
 * the payload bytes blockSearch would ReadAt (block_search.go:411-474). */
typedef struct vlscan_column {
    uint32_t field;         /* index into the batch's field-name table                                             */
    uint8_t kind;           /* VLSCAN_COL_*                                                                        */
    uint8_t value_type;     /* VLSCAN_VT_* (VALUES only)                                                           */
    uint8_t stage;          /* VLSCAN_STAGE_* (VALUES only)                                                        */
    uint8_t dict_len;       /* number of valuesDict entries (<= 8, values_encoder.go:1243-1322)                    */
    uint64_t min_value;     /* columnHeader.minValue / maxValue (raw u64 bits; meaning depends on value_type)      */
    uint64_t max_value;
    const uint8_t* const_value; uint64_t const_len;      /* CONST: the value (<= 256 B, consts.go:41)              */
    const uint8_t* dict_blob;   const uint32_t* dict_offsets; /* DICT: concatenated values + dict_len+1 offsets     */
    const uint8_t* values;      uint64_t values_len;     /* STAGE_ONDISK                                           */
    const uint8_t* lens_items;  uint64_t lens_items_len; /* STAGE_DECODED                                          */
    const uint8_t* data;        uint64_t data_len;       /* STAGE_DECODED                                          */
    const uint8_t* bloom;       uint64_t bloom_len;      /* big-endian u64 words as stored (bloomfilter.go:49-71)  */
} vlscan_column;

/* One block = blockSearchWork.bh.rowsCount + the columns the program references (block_search.go:64-77), and optionally its timestamps
 * column: the bytes at [timestampsHeader.blockOffset, +blockSize) of timestamps.bin as stored (encoding.MarshalTimestamps with
 * precisionBits = 64, lib/logstorage/block.go:674-690) plus the three header fields UnmarshalTimestamps needs (block_header.go:990-997).
 * ZSTD marshal types are inflated on the device like values blocks.  Timestamps are needed by `_time` filters that only partly overlap
 * the block (filter_time.go:114-137) and by vlscan_gather_timestamps; blocks handed over without them fail such a scan with an error. */
typedef struct vlscan_block {
    uint64_t rows;
    uint32_t ncols;
    uint32_t ts_marshal_type;         /* 0 = no timestamps given; else encoding.MarshalType 1..6 (vm/lib/encoding/encoding.go:20-43) */
    const vlscan_column* cols;
    const uint8_t* timestamps; uint64_t timestamps_len;
    int64_t min_timestamp, max_timestamp;   /* timestampsHeader.minTimestamp (= the first row's timestamp) and maxTimestamp */
} vlscan_block;

/* Counters of one scan (block_stats-like accounting, lib/logstorage/pipe_block_stats.go:90-105). Algorithmic bytes
 * are block-granular and follow the reference's short-circuit order (a column is charged when the reference would
 * have called getValuesForColumn / getBloomFilterForColumn for it). */
typedef struct vlscan_stats {
    uint64_t blocks;              /* blocks submitted                                                              */
    uint64_t rows;                /* rows submitted ("rows scanned")                                               */
    uint64_t rows_matched;        /* sum of popcounts                                                              */
    uint64_t blocks_matched;      /* blocks with a non-zero bitmap                                                 */
    uint64_t values_bytes;        /* decoded payload (lens items + data) of every column read                      */
    uint64_t bloom_probe_bytes;   /* 8 B x probes                                                                  */
    uint64_t bitmap_bytes;        /* 8 B x words of non-zero result bitmaps                                        */
    uint64_t columns_read;        /* (block, column) pairs whose values were read                                  */
    uint64_t gpu_launches;        /* kernels launched by this call                                                 */
    uint64_t h2d_bytes;           /* host->device bytes moved by this call                                         */
    uint64_t d2h_bytes;           /* device->host bytes moved by this call                                         */
    double gpu_ms;                /* device time of the scan kernels (CUDA events on the ctx stream)               */
    double scan_kernel_ms;        /* device time of the dominant string-scan kernel launches only                  */
    uint64_t scan_kernel_bytes;   /* algorithmic bytes processed by those launches                                 */
    uint64_t staged_columns;      /* vlscan_scan_batch, bloom-first staging: (block, column) values payloads uploaded ...          */
    uint64_t pruned_columns;      /* ... and left on the host because no filter could reach them (0 / 0 when staged in one go)     */
} vlscan_stats;

/* Synthetic data set description (benchmark / test infrastructure; row shape of app/vlogsgenerator/main.go:240-281). */
typedef struct vlscan_gen_config {
    uint64_t seed;
    uint64_t total_rows;
    uint32_t rows_per_block;
    uint32_t hot_block_permille;
    uint32_t hit_row_permille;
    uint32_t columns_mask;       /* bit0 _msg, bit1 level, bit2 path, bit3 status; bit4 a timestamps column: row i of the data set at
                                    VLSCAN_GEN_T0 + i ms (MarshalTypeDeltaConst); bits 8..11: vocabulary focus for selectivity sweeps
                                    (0 = a vocabulary row draws one of the 12 entries uniformly, k = always entry k - 1); bits 12..16,
                                    only together with bit 4: k <= 16, S = 2^k blocks interleave in time: row i of block b at
                                    VLSCAN_GEN_T0 + ((b / S) * S * rows_per_block + i * S + b % S) ms, still DeltaConst (k = 0: as bit 4
                                    alone) */
} vlscan_gen_config;
#define VLSCAN_GEN_T0 1700000000000000000ll   /* 2023-11-14T22:13:20Z, nanoseconds */
#define VLSCAN_GEN_STEP 1000000ll            /* 1 ms between consecutive rows */

/* ---- library / worker context ---------------------------------------------------------------------------------- */
int vlscan_device_count(void);                               /* number of usable CUDA devices (0 => nothing works)  */
vlscan_ctx* vlscan_ctx_create(int device);                   /* replaces getBlockSearch() per worker
                                                                (storage_search.go:1041-1043); NULL on failure     */
void vlscan_ctx_free(vlscan_ctx* ctx);
const char* vlscan_last_error(const vlscan_ctx* ctx);        /* ctx may be NULL: last error of the calling thread   */
void* vlscan_ctx_stream(const vlscan_ctx* ctx);              /* the cudaStream_t all work of this ctx is issued on  */
int vlscan_ctx_sync(vlscan_ctx* ctx);                        /* cudaStreamSynchronize                               */

/* ---- program: the filter tree ---------------------------------------------------------------------------------- */
/* `tree` is the filter tree serialised depth-first (the Go shim walks `filter` values, lib/logstorage/filter.go:8-20):
 *   node   := kind:u8 payload
 *   bytes  := varuint(len) raw            (vm/encoding/int.go:506-527 MarshalBytes)
 *   0 NOOP    (filter_noop.go)            -
 *   1 PHRASE  (filter_phrase.go:25-32)    bytes(fieldName) bytes(phrase)
 *   2 PREFIX  (filter_prefix.go:20-27)    bytes(fieldName) bytes(prefix)
 *   3 EXACT   (filter_exact.go:17-24)     bytes(fieldName) bytes(value)
 *   4 IN      (filter_in.go:14-18)        bytes(fieldName) varuint(n) n x bytes(value)
 *   5 REGEXP  (filter_regexp.go:17-24)    bytes(fieldName) bytes(regexp source, regexutil.Regex.String())
 *   6 AND     (filter_and.go:15-20)       varuint(n) n x node
 *   7 OR      (filter_or.go:36-41)        varuint(n) n x node
 *   8 NOT     (filter_not.go:11-13)       node
 *   9 EXACT_PREFIX (filter_exact_prefix.go:13-20)   bytes(fieldName) bytes(prefix)                         `f:="abc"*`
 *  10 LEN_RANGE    (filter_len_range.go:14-22)      bytes(fieldName) varuint(minLen) varuint(maxLen)        `f:len_range(a, b)`
 *  11 STRING_RANGE (filter_string_range.go:12-20)   bytes(fieldName) bytes(minValue) bytes(maxValue)        `f:string_range(a, b)`, [min, max)
 *  12 IPV4_RANGE   (filter_ipv4_range.go:12-20)     bytes(fieldName) varuint(minValue) varuint(maxValue)    `f:ipv4_range(a, b)`, inclusive
 *  13 VALUE_TYPE   (filter_value_type.go:12-15)     bytes(fieldName) bytes(type name)                       `f:value_type(uint8)`
 *  14 ANY_CASE_PHRASE (filter_any_case_phrase.go:14-24)   bytes(fieldName) bytes(phrase as written)            `f:i(phrase)`
 *  15 ANY_CASE_PREFIX (filter_any_case_prefix.go:14-24)   bytes(fieldName) bytes(prefix as written)            `f:i(prefix*)`
 *  16 SEQUENCE     (filter_sequence.go:12-22)       bytes(fieldName) varuint(n) n x bytes(phrase)           `f:seq(a, b, ...)`
 *  17 CONTAINS_ALL (filter_contains_all.go:12-20)   bytes(fieldName) varuint(n) n x bytes(value)            `f:contains_all(a, b, ...)`
 *  18 CONTAINS_ANY (filter_contains_any.go:12-20)   bytes(fieldName) varuint(n) n x bytes(value)            `f:contains_any(a, b, ...)`
 *  19 EQ_FIELD     (filter_eq_field.go:14-22)       bytes(fieldName) bytes(otherFieldName)                  `f:eq_field(g)`
 *  20 LE_FIELD     (filter_le_field.go:14-24)       bytes(fieldName) bytes(otherFieldName) u8(excludeEqualValues)   `f:le_field(g)`, `f:lt_field(g)`
 *  21 RANGE        (filter_range.go:14-24)          bytes(fieldName) f64le(minValue) f64le(maxValue)        `f:range[a, b]`, `f:>a`, `f:<=b` ...
 *  22 TIME         (filter_time.go:14-23)           i64le(minTimestamp) i64le(maxTimestamp)                 `_time:[a, b]`, nanoseconds, inclusive
 * Token hashes, merged AND/OR per-field tokens, typed needles and regex automata are derived here, like the
 * sync.Once initialisers of the Go filters do on first use.  Returns <0 with an error text for malformed trees,
 * regexps that do not compile and regexps outside the supported syntax. */
enum { VLSCAN_F_NOOP = 0, VLSCAN_F_PHRASE, VLSCAN_F_PREFIX, VLSCAN_F_EXACT, VLSCAN_F_IN, VLSCAN_F_REGEXP, VLSCAN_F_AND, VLSCAN_F_OR, VLSCAN_F_NOT,
       VLSCAN_F_EXACT_PREFIX = 9, VLSCAN_F_LEN_RANGE = 10, VLSCAN_F_STRING_RANGE = 11, VLSCAN_F_IPV4_RANGE = 12, VLSCAN_F_VALUE_TYPE = 13,
       VLSCAN_F_ANY_CASE_PHRASE = 14, VLSCAN_F_ANY_CASE_PREFIX = 15, VLSCAN_F_SEQUENCE = 16, VLSCAN_F_CONTAINS_ALL = 17, VLSCAN_F_CONTAINS_ANY = 18, VLSCAN_F_EQ_FIELD = 19, VLSCAN_F_LE_FIELD = 20, VLSCAN_F_RANGE = 21, VLSCAN_F_TIME = 22 };
int vlscan_program_create(const void* tree, size_t tree_len, vlscan_program** out);
void vlscan_program_free(vlscan_program* prog);
/* canonical names of the fields the tree references (so the caller lists only those columns per block) */
uint32_t vlscan_program_nfields(const vlscan_program* prog);
const char* vlscan_program_field(const vlscan_program* prog, uint32_t i, size_t* len);
/* token strings of a leaf (tests; mirrors filterPhrase.getTokens() etc.), '\n'-joined into buf; returns length or -1 */
int64_t vlscan_program_leaf_tokens(const vlscan_program* prog, uint32_t leaf, char* buf, size_t cap);
/* the per-field tokens of the bloom pre-pass of every AND / OR node (filterAnd.byFieldTokens filter_and.go:122-187, filterOr.byFieldTokens
 * filter_or.go:126-193), nodes in pre-order, one line each: "A" or "O", then per field "\t" field "\x1f" token "\x1f" token ...; returns the
 * length or -1 when cap is too small.  For tests against the oracle. */
int64_t vlscan_program_prepass_tokens(const vlscan_program* prog, char* buf, size_t cap);
/* the bloom probe hashes of an in() leaf (inValues.getTokensHashesAny, in_values.go:104-140,317-371): out = n_common, the common hashes,
 * n_sets (UINT64_MAX when there are more than maxTokenSetsToInit = 1000 values and no set is kept), then per value set: n, hashes.
 * Returns the number of u64 written, -1 when the leaf is not an in() or cap is too small.  For tests against the oracle. */
int64_t vlscan_program_in_hashes(const vlscan_program* prog, uint32_t leaf, uint64_t* out, size_t cap);
/* the sorted typed value set an in() leaf is matched with on a column of `value_type` (inValues.getUint8Values ... getTimestampISO8601Values,
 * in_values.go:141-315): uintN / ipv4 as numbers, int64 zig-zag coded, float64 as bits, iso8601 as nanoseconds.  Returns the count or -1. */
int64_t vlscan_program_in_typed(const vlscan_program* prog, uint32_t leaf, int value_type, uint64_t* out, size_t cap);
/* text of a float64 column value as the filters see it: marshalFloat64String (values_encoder.go:1397-1399), i.e.
 * strconv.AppendFloat(f, 'f', -1, 64).  Host build of the routine the scan kernels run per row; returns the length
 * (<= 344) or -1 when cap is too small.  No NUL terminator is written. */
int vlscan_format_float64(uint64_t ieee_bits, char* buf, size_t cap);
/* parseMathNumber (lib/logstorage/pipe_math.go:1066-1080): the number a string value stands for in range(), le_field() and lt_field() - plain and
 * `_`-separated decimals, durations ("1h5m"), byte sizes ("10KiB"), Go number literals (exponents, hexadecimal floats, base prefixes, inf), RFC 3339
 * timestamps (nanoseconds; UTC where the text names no zone) and IPv4 addresses - or NaN.  Host build of the routine the row kernels run per
 * value (csrc/vl_mathnum.cuh; decimal -> double is correctly rounded).  For tests against the oracle. */
double vlscan_parse_math_number(const void* s, size_t len);
/* how the program compiler reads a filter argument as a value of a typed column (tryParseUint64 / tryParseInt64 / tryParseFloat64Exact /
 * tryParseIPv4 / tryParseTimestampISO8601, values_encoder.go:428-850): 1 and *out = the value (int64 and float64 as their bits) when the text
 * is one, 0 when it is not, -1 for value types without a typed form.  For tests against the oracle. */
int vlscan_parse_typed(int value_type, const void* s, size_t len, uint64_t* out);
/* Host build of the per-value predicate the row kernels run for filter kinds 9..12 (matchExactPrefix, matchLenRange,
 * matchStringRange, matchIPv4Range): arg1 = prefix / minValue, arg2 = maxValue, aux0..aux1 = minLen..maxLen or the IPv4
 * bounds.  Returns 1 / 0, or -1 for other kinds.  For tests against the oracle.
 * kind 5 (REGEXP): arg1 = the expression; compiled like a regexp leaf and matched by the host mirror of the device automaton (the
 * form const and dict values are matched with); -2 when the expression does not compile.
 * Also answers for the value predicates of kinds 14..18 (host builds of the host+device code in csrc/vl_anycase.cuh):
 * 14 = matchAnyCasePhrase, 15 = matchAnyCasePrefix (arg1 = the phrase / prefix already lowercased by
 * strings.ToLower), 16 = matchSequence, 17 = matchAllPhrases, 18 = matchAnyPhrase (arg1 = phrase list, each as varuint length + bytes). */
int vlscan_eval_predicate(int kind, const void* value, size_t value_len, const void* arg1, size_t arg1_len, const void* arg2,
                          size_t arg2_len, uint64_t aux0, uint64_t aux1);

/* ---- batches ---------------------------------------------------------------------------------------------------- */
/* Stage `nblocks` blocks into HBM (host pointers in, pinned staging + cudaMemcpyAsync inside).  Field names are the
 * canonical column names ("_msg" for the empty name, getCanonicalColumnName). */
int vlscan_batch_upload(vlscan_ctx* ctx, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields,
                        const vlscan_block* blocks, uint64_t nblocks, vlscan_batch** out, vlscan_stats* stats /* may be NULL: h2d_bytes */);
void vlscan_batch_free(vlscan_batch* batch);
uint64_t vlscan_batch_nblocks(const vlscan_batch* batch);
uint64_t vlscan_batch_rows(const vlscan_batch* batch);
uint64_t vlscan_batch_words(const vlscan_batch* batch);      /* sum over blocks of ceil(rows/64)                    */
uint64_t vlscan_batch_device_bytes(const vlscan_batch* batch);

/* Generate blocks [block_lo, block_hi) of a synthetic data set directly in HBM (decoded stage + bloom filters, byte-
 * identical to what the reference writer path would produce for the same rows; verified against the oracle). */
int vlscan_batch_generate(vlscan_ctx* ctx, const vlscan_gen_config* cfg, uint64_t block_lo, uint64_t block_hi, vlscan_batch** out);

/* Copy a resident batch back into caller-visible host memory as vlscan_block descriptors (decoded stage, timestamps columns in their plain
 * marshal types).  The
 * descriptors and payloads live in one library-owned pinned host buffer that stays valid until vlscan_host_blocks_free. */
typedef struct vlscan_host_blocks vlscan_host_blocks;
int vlscan_batch_download(vlscan_ctx* ctx, const vlscan_batch* batch, vlscan_host_blocks** out);
const vlscan_block* vlscan_host_blocks_get(const vlscan_host_blocks* hb, uint64_t* nblocks, uint32_t* nfields);
const char* vlscan_host_blocks_field(const vlscan_host_blocks* hb, uint32_t i, size_t* len);
uint64_t vlscan_host_blocks_bytes(const vlscan_host_blocks* hb);
void vlscan_host_blocks_free(vlscan_host_blocks* hb);
/* Writer-side helper for benches and tests: re-encode the values blocks of `in` into their on-disk form,
 * marshalBytesBlock(lens items) ++ marshalBytesBlock(data) with the reference's size-dependent ZSTD level
 * (lib/logstorage/encoding.go:16-50,343-370), using libzstd on `threads` host threads (0 = all).  The result lives in one
 * pinned buffer whose layout lets vlscan_batch_upload / vlscan_scan_batch move it with two DMA transfers.
 * Compression is the only thing libzstd is used for; frames are decoded on the device. */
int vlscan_host_blocks_compress(const vlscan_host_blocks* in, int threads, vlscan_host_blocks** out);

/* ---- device ZSTD decoder --------------------------------------------------------------------------------------------
 * VLSCAN_STAGE_ONDISK payloads are copied to HBM compressed and regenerated there (replaces the libzstd call behind
 * unmarshalBytesBlock, encoding.go:372-426 -> lib/encoding/compress.go:24-32).  This entry point runs the same decoder on
 * `nframes` independent frames given as host pointers, for parity tests against libzstd: frame i must regenerate exactly
 * dst_offsets[i+1]-dst_offsets[i] bytes, written to dst + dst_offsets[i].  Frames must declare their content size and use
 * no dictionary; content checksums are skipped, not verified. */
int vlscan_zstd_decompress(vlscan_ctx* ctx, uint32_t nframes, const void* const* frames, const size_t* frame_lens, void* dst,
                           const uint64_t* dst_offsets);
/* The host half of that decoder alone (no device needed): walk ONE bytes block (marshalBytesBlock container, encoding.go:343-360)
 * exactly like the stager does - container, frame header, block headers, literals / sequences section headers - and report
 * out[0] = bytes consumed, out[1] = regenerated length, out[2] = ZSTD blocks, out[3] = compressed blocks, out[4] = sequences.
 * Returns <0 with an error text for malformed input.  For tests (the walker parses untrusted bytes). */
int vlscan_zstd_inspect(const void* bytes_block, size_t len, uint64_t out[5]);
/* The same walk over every VLSCAN_STAGE_ONDISK column of `nblocks` blocks, as vlscan_batch_upload / vlscan_scan_batch run it, on
 * `threads` host threads (0: one block after the other on the calling thread; uploads use $VLSCAN_HOST_THREADS, default min(16, cores)).
 * out[0..3] = digest of everything the walk hands to the device (frame table, ZSTD block table with scratch offsets and table slots,
 * launch groups, work lists): the same for every thread count.  out[4] = frames, out[5] = ZSTD blocks, out[6] = launch groups,
 * out[7] = compressed blocks, out[8] = sequences, out[9] / out[10] = nanoseconds spent walking / building the work lists, out[11] = 0.
 * No device needed.  For tests and host-side tuning. */
int vlscan_zstd_walk_digest(const vlscan_block* blocks, uint64_t nblocks, int threads, uint64_t out[12]);

/* ---- part directory reader -----------------------------------------------------------------------------------------
 * For hosts without the Go process: opens one part directory the way part.mustOpenFilePart does (lib/logstorage/part.go:105-173;
 * format versions 1..3) and hands out, for any block range and field list, the vlscan_block descriptors (VLSCAN_STAGE_ONDISK, pointing
 * into the memory-mapped bloom / values files) that vlscan_scan_batch and vlscan_batch_upload take - what blockSearch.getColumnHeader /
 * getConstColumnValue / getBloomFilterForColumn / getValuesForColumn (block_search.go:232-474) locate lazily per block.
 * The part's own ZSTD-compressed metadata (column_names.bin, metaindex.bin, the blocks of index.bin: a few KB..MB) is inflated by the
 * device decoder of `ctx`, or, when the embedding process has its own ZSTD (the Go process does), by `inflate`: it must regenerate
 * exactly dst_len bytes from the frame and return 0.  Values blocks never go through `inflate`. */
typedef struct vlscan_part vlscan_part;
typedef int (*vlscan_inflate_fn)(void* user, const void* frame, size_t frame_len, void* dst, size_t dst_len);
int vlscan_part_open(vlscan_ctx* ctx /* may be NULL with inflate */, const char* path, vlscan_inflate_fn inflate /* may be NULL with ctx */, void* user, vlscan_part** out);
void vlscan_part_free(vlscan_part* part);
/* partHeader (metadata.json): FormatVersion, CompressedSizeBytes, UncompressedSizeBytes, RowsCount, BlocksCount, MinTimestamp, MaxTimestamp,
 * BloomValuesShardsCount */
void vlscan_part_header(const vlscan_part* part, uint64_t out[8]);
uint64_t vlscan_part_nblocks(const vlscan_part* part);
/* blockHeader i in index order (streamID, then minTimestamp): accountID, projectID, streamID.hi, streamID.lo, uncompressedSizeBytes, rowsCount,
 * timestamps blockOffset, blockSize, minTimestamp, maxTimestamp, marshalType, columnsHeaderIndexOffset, -Size, columnsHeaderOffset, -Size */
int vlscan_part_block_header(const vlscan_part* part, uint64_t i, uint64_t out[15]);
/* the encoded timestamps of block i as stored in timestamps.bin (encoding.MarshalTimestamps; marshalType, first value = minTimestamp and
 * rowsCount are in the block header): for the rows of blocks that only partly overlap a time range, until the engine filters _time itself */
int vlscan_part_timestamps(const vlscan_part* part, uint64_t i, const uint8_t** data, uint64_t* len);
uint32_t vlscan_part_ncolumn_names(const vlscan_part* part);
const char* vlscan_part_column_name(const vlscan_part* part, uint32_t i, size_t* len);   /* "" is the message field */
/* Descriptors of the blocks [block_lo, block_hi) whose [minTimestamp, maxTimestamp] overlaps [min_timestamp, max_timestamp], restricted to
 * the given fields ("_msg" or "" = the message field); a field a block does not have is simply absent from it.  The result stays valid
 * while the part is open; vlscan_host_blocks_source tells which block of the part each described block is. */
int vlscan_part_blocks(const vlscan_part* part, const char* const* field_names, const size_t* field_name_lens, uint32_t nfields, uint64_t block_lo,
                       uint64_t block_hi, int64_t min_timestamp, int64_t max_timestamp, vlscan_host_blocks** out);
const uint64_t* vlscan_host_blocks_source(const vlscan_host_blocks* hb, uint64_t* n);

/* ---- the scan ---------------------------------------------------------------------------------------------------- */
/* Scan a resident batch: equivalent of `for each block: bm.init(rows); bm.setBits(); filter.applyToBlockSearch(bs, bm)`
 * (block_search.go:207-215).  Results stay on the device until fetched; the call only enqueues work on the ctx stream
 * (no host synchronisation) unless `stats` is non-NULL, in which case it synchronises and fills the counters. */
int vlscan_scan_resident(vlscan_ctx* ctx, const vlscan_program* prog, const vlscan_batch* batch, vlscan_stats* stats);

/* Counters + device timings of the most recent vlscan_scan_resident on this ctx (synchronises the ctx stream). */
int vlscan_last_scan_stats(vlscan_ctx* ctx, vlscan_stats* stats);

/* Fetch the results of the last vlscan_scan_resident on this ctx.
 *   out_bitmap_words : packed per-block bitmaps, block b at word offset sum_{i<b} ceil(rows_i/64); bit i%64 of word i/64
 *                      = row i, tail bits zero (lib/logstorage/bitmap.go:28-31,62-72) so Go can alias it as bitmap.a
 *   out_match_counts : per block onesCount() (bitmap.go:185-191) == blockResult.rowsLen (block_result.go:403-414)
 * Either may be NULL. Synchronises the ctx stream.  Bitmaps and counts live in the ctx: the scanned batch may already have been freed. */
int vlscan_fetch_results(vlscan_ctx* ctx, uint64_t* out_bitmap_words, uint32_t* out_match_counts, vlscan_stats* stats /* may be NULL: d2h_bytes */);
/* Ascending hit-row indexes (u32 per hit, row index within its block) of the last scan, block after block; for callers
 * that want to skip forEachSetBitReadonly (bitmap.go:156-183).  out_hit_offsets has nblocks+1 entries. */
int vlscan_fetch_hits(vlscan_ctx* ctx, uint32_t* out_hit_rows, uint64_t cap, uint64_t* out_hit_offsets);
/* ---- hit materialisation: what blockResult reads for the selected rows (lib/logstorage/block_result.go:491-507, 529-591) -----------------------
 * Both calls work on the result of the last vlscan_scan_resident of this ctx; its batch must still be alive.  Hits are ordered block after block,
 * rows ascending (the order of vlscan_fetch_hits); out_hit_offsets (nblocks + 1 entries, may be NULL) receives the first hit of every block.
 *
 * vlscan_gather_timestamps: the `_time` of every selected row (blockResult.initTimestampsInternal): the timestamps blocks of the blocks with hits
 *   are decoded on the device (encoding.UnmarshalTimestamps, all marshal types).  The batch must have been staged with timestamps.
 * vlscan_gather_values: the value of `field` in every selected row as a string, the way blockResultColumn.getValues yields it: row bytes of a
 *   strings column, the dictionary entry of a dict column, the text form of a typed value (marshalUint64String ... marshalTimestampISO8601String,
 *   values_encoder.go:1367-1422), the value of a const column, "" for a field the block does not have.  out_value_offsets gets hits + 1 entries
 *   (cap_values >= hits); the bytes of hit h are out_bytes[offsets[h], offsets[h + 1]).  *out_total_bytes = bytes needed, also when the call fails
 *   because cap_bytes is too small (then nothing is written to out_bytes). */
int vlscan_gather_timestamps(vlscan_ctx* ctx, int64_t* out_timestamps, uint64_t cap, uint64_t* out_hit_offsets);
int vlscan_gather_values(vlscan_ctx* ctx, const char* field, size_t field_len, uint8_t* out_bytes, uint64_t cap_bytes, uint64_t* out_value_offsets, uint64_t cap_values,
                         uint64_t* out_total_bytes, uint64_t* out_hit_offsets);
/* ---- the hits histogram: `stats by (_time:step offset off, f1, ...) count() hits` over the selected rows of the last scan ------------------------
 * The aggregation /select/logsql/hits appends to every query (app/vlselect/logsql/logsql.go:116-219, lib/logstorage/parser.go:407-445), computed
 * on the device so that only the groups cross PCIe.  Same preconditions as the gather calls: the result of the last vlscan_scan_resident of the
 * ctx, whose batch must still be alive.  Every block with selected rows must have been staged with its timestamps.
 *   bucket of a row: truncateTimestamp (lib/logstorage/block_result.go:818-848); step = int64(byStatsField.bucketSize) (<= 0 counts as 1),
 *     offset = int64(bucketOffset), both in nanoseconds; calendar = VLSCAN_BUCKET_WEEK / _MONTH / _YEAR when bucketSizeStr is "week" / "month" /
 *     "year" (the week starts on Monday; month and year are UTC calendar units, step is then ignored), VLSCAN_BUCKET_PLAIN otherwise (the
 *     /hits endpoint always: its step is a duration such as "1w").  int64 arithmetic wraps like Go's.
 *   group key: the bucket, then the text of every by-field as vlscan_gather_values yields it (typed values formatted, "" for a field a block does
 *     not have): `200` stored as uint16 in one block and as a string in another is one group.  Keys are compared byte for byte, never by hash.
 *   by_names: canonical field names ("" = _msg), at most VLSCAN_HITS_MAX_BY; "_time" is rejected.  by_names and by_name_lens may be NULL only when nby == 0.
 *   by_buckets (vlscan_hits_stats_bucketed / vlscan_hits_sums_bucketed; NULL: no by-field has a bucket, the call is vlscan_hits_stats /
 *     vlscan_hits_sums): `stats by (f:size offset off)`, one entry per by-field, filled from byStatsField: size =
 *     bucketSize, offset = bucketOffset, calendar = VLSCAN_BUCKET_* of bucketSizeStr (week / month / year; month and year leave size 0),
 *     enabled = hasBucketConfig().  An enabled by-field keys on its bucketed text (newValuesBucketedForColumn, lib/logstorage/block_result.go:703-1764):
 *       const value, string row, dict entry   getBucketedValue(text): "" and a text that does not start with 0-9 or '-' stay as they are; else
 *                                             the first of tryParseInt64 (truncateInt64, int64 text), tryParseFloat64 (truncateFloat64,
 *                                             marshalFloat64String), TryParseTimestampRFC3339Nano (truncateTimestamp, RFC3339Nano),
 *                                             tryParseIPv4 (truncateUint32, IPv4 text), tryParseDuration (truncateInt64, marshalDurationString)
 *                                             that accepts it; a text none accepts stays as it is
 *       uint8 .. uint64                       truncateUint64(n, uint64(size), uint64(int64(offset))) -> decimal
 *       int64                                 truncateInt64(n, int64(size), int64(offset)), a size of 0 counting as 1 -> decimal
 *       float64                               truncateFloat64(f, p10, int64(size * p10), offset), p10 = math.Pow10(-e), e the exponent of
 *                                             decimal.FromFloat(size) -> marshalFloat64String
 *       ipv4                                  truncateUint32(n, uint32(size), uint32(int32(offset))) -> IPv4 text
 *       iso8601                               truncateTimestamp(ts, int64(size), int64(offset), calendar) -> ISO 8601 text
 *     Unsigned sizes of 0 and signed sizes <= 0 count as 1 except where noted; float -> integer conversions are Go's on amd64.  A typed column
 *     whose header minimum and maximum fall into one bucket gives every row of its block that bucket (for float64 also when rows are NaN).  A
 *     bucketed by-field a block lacks is "".  Keys compare bucketed texts byte for byte: `200` stored as uint16 and `250` as a string are one
 *     group under size 100.  A NaN or infinite size or offset, an unknown calendar and a size whose int64(size * p10) is 0 (the reference
 *     would divide by zero) fail the call.
 * Output: the groups sorted by bucket, then by the key texts bytewise: out_buckets[g], out_counts[g] (rows), and the texts of group g's by-field
 * f at out_key_bytes[out_key_offsets[g * nby + f], out_key_offsets[g * nby + f + 1]) (out_key_offsets has cap_groups * nby + 1 entries).
 * out_info (may be NULL) = {groups, key bytes, selected rows, blocks whose timestamps were decoded}; it is filled also when the call fails because
 * cap_groups or cap_key_bytes is too small (then nothing else is written).  Blocks whose minimum and maximum timestamps fall into one bucket
 * are counted without decoding their timestamps. */
enum { VLSCAN_BUCKET_PLAIN = 0, VLSCAN_BUCKET_WEEK = 1, VLSCAN_BUCKET_MONTH = 2, VLSCAN_BUCKET_YEAR = 3 };
#define VLSCAN_HITS_MAX_BY 4
typedef struct vlscan_by_bucket {
    double size, offset;           /* byStatsField.bucketSize, bucketOffset                                                       */
    uint32_t calendar;             /* VLSCAN_BUCKET_*                                                                             */
    uint32_t enabled;              /* byStatsField.hasBucketConfig()                                                              */
} vlscan_by_bucket;
typedef struct vlscan_hits_query {
    int64_t step, offset;          /* nanoseconds */
    uint32_t calendar;             /* VLSCAN_BUCKET_*                                                                             */
    uint32_t nby;                  /* by-fields after _time, <= VLSCAN_HITS_MAX_BY                                                */
    const char* const* by_names;
    const size_t* by_name_lens;
} vlscan_hits_query;
int vlscan_hits_stats(vlscan_ctx* ctx, const vlscan_hits_query* q, int64_t* out_buckets, uint64_t* out_counts, uint64_t cap_groups, uint8_t* out_key_bytes,
                      uint64_t cap_key_bytes, uint64_t* out_key_offsets, uint64_t out_info[4]);
/* vlscan_hits_stats with by_buckets: q->nby entries, or NULL */
int vlscan_hits_stats_bucketed(vlscan_ctx* ctx, const vlscan_hits_query* q, const vlscan_by_bucket* by_buckets, int64_t* out_buckets, uint64_t* out_counts,
                               uint64_t cap_groups, uint8_t* out_key_bytes, uint64_t cap_key_bytes, uint64_t* out_key_offsets, uint64_t out_info[4]);
/* ---- `stats by (_time:step offset off, f1, ...) count(), sum(v1), avg(v1), ...` over the selected rows of the last scan --------------------------
 * The grouping of vlscan_hits_stats (same query, same preconditions, same groups in the same order with the same keys and row counts) plus, per
 * group g and value field f, the partial state a stats shard exports for sum(f) and avg(f) (lib/logstorage/stats_sum.go, stats_avg.go):
 *   out_value_counts[g * nvalues + f]: how many numbers the field gave (statsAvgProcessor.count);
 *   out_sums[g * nvalues + f]: their sum, NaN when the count is 0 (statsSumProcessor.sum; avg's sum is the same number with 0 for NaN).
 * The numbers of a block come from blockResultColumn.sumValues when every selected row of the block has one group key, else from
 * getFloatValueAtRow row by row (pipe_stats.go:552-626, 700-730).  The two differ: sumValues parses strings and dict entries with tryParseNumber
 * (durations, byte sizes: "1KiB", "5s") and counts every row of a float64 column, getFloatValueAtRow parses them with tryParseFloat64 and skips
 * NaN float64 rows.  Both parse a const value with tryParseFloat64, read uint8..uint64 / int64 as float64(v), and take nothing from ipv4 /
 * iso8601 columns, `_time` or a field a block lacks.
 * A sum is the exact sum of the numbers (each cut to 92 bits below the largest of its group), rounded once: integer inputs whose sum stays below
 * 2^53 give it exactly, and the result does not depend on the order of rows or blocks.  A group with both +Inf and -Inf, or a NaN number, sums
 * to NaN (the reference's float adds there depend on row order).
 *   value_names: canonical names ("" = _msg), 1 ..VLSCAN_STATS_MAX_VALUES of them; a name ending in `*` (a prefix filter such as `sum(foo*)`) is rejected.  On a
 *   kept batch the values of every value field must have been staged in every block with selected rows (the error names the field).
 * The caller merges batches per group key: rows and counts add, sums add with NaN as "none" (victorialogs_b200.scan.stats_merge). */
#define VLSCAN_STATS_MAX_VALUES 4
int vlscan_hits_sums(vlscan_ctx* ctx, const vlscan_hits_query* q, const char* const* value_names, const size_t* value_name_lens, uint32_t nvalues, int64_t* out_buckets,
                     uint64_t* out_counts, double* out_sums, uint64_t* out_value_counts, uint64_t cap_groups, uint8_t* out_key_bytes, uint64_t cap_key_bytes,
                     uint64_t* out_key_offsets, uint64_t out_info[4]);
/* vlscan_hits_sums with by_buckets: q->nby entries, or NULL.  The sums follow the bucketed keys: a block whose raw values differ but fall into
 * one bucket is one group, added through sumValues. */
int vlscan_hits_sums_bucketed(vlscan_ctx* ctx, const vlscan_hits_query* q, const vlscan_by_bucket* by_buckets, const char* const* value_names,
                              const size_t* value_name_lens, uint32_t nvalues, int64_t* out_buckets, uint64_t* out_counts, double* out_sums,
                              uint64_t* out_value_counts, uint64_t cap_groups, uint8_t* out_key_bytes, uint64_t cap_key_bytes, uint64_t* out_key_offsets,
                              uint64_t out_info[4]);
/* The bucket of one timestamp: host build of the routine the hits kernels run per row (truncateTimestamp above).  For tests. */
int64_t vlscan_truncate_timestamp(int64_t ts, int64_t step, int64_t offset, uint32_t calendar);
/* The bucketed text of one const, string or dict text s under bucket b (getBucketedValue above): host build of the routine the hits kernels run.
 * Returns its length (<= 352; no NUL written), -1 when cap is too small, -2 for a bucket vlscan_hits_stats rejects.  b->enabled is ignored.  For tests. */
int vlscan_bucket_text(const vlscan_by_bucket* b, const void* s, size_t len, char* out, size_t cap);
/* ---- `stats by (_time:step offset off, f1, ...) histogram(v...)` (lib/logstorage/stats_histogram.go) --------------------------------------------
 * Per group and value field, the numbers counted per vmrange bucket of metrics.Histogram (VictoriaMetrics/metrics histogram.go).  Groups, keys,
 * rows, their order, by_buckets, value_names and the preconditions and errors are those of vlscan_hits_sums_bucketed (a trailing `*` is rejected:
 * `histogram(a*)` does not parse).  A number is what both stats_histogram.go paths read: tryParseNumber of a const, string or dict text
 * (durations, byte sizes, 0x..., 1_000; "" is none), float64(n) of a uint8..uint64 / int64 row, the double of a float64 row; ipv4 and iso8601
 * rows, a field the block lacks and `_time` give none.  Histogram.Update then skips NaN and v < 0 (not -0) and indexes the rest:
 *   index 0 = "0...1.000e-09" (Log10(v) + 9 < 0, -0 and +0 included), 1 .. 486 = metrics bucket index + 1, 487 = "1.000e+18...+Inf" (1e18 and +Inf
 *   included).  Index order is numeric order; vlscan_vmrange_text gives the vmrange text of an index.
 * Entries: those of (group g, value field f) are out_entry_ranges / out_entry_hits [out_entry_offsets[g * nvalues + f] .. [+ 1]), non-zero
 * counts only, by ascending index; out_entry_offsets has cap_groups * nvalues + 1 items.  out_info = {groups, key bytes, selected rows, blocks
 * whose timestamps were decoded, entries, (block, value field) cells counted from their column header alone}, filled also when a capacity is too
 * small.  The caller merges batches per (group key, value field, index): hits add (victorialogs_b200.scan.vmranges_merge). */
#define VLSCAN_VMRANGES 488
int vlscan_hits_vmranges(vlscan_ctx* ctx, const vlscan_hits_query* q, const vlscan_by_bucket* by_buckets, const char* const* value_names,
                         const size_t* value_name_lens, uint32_t nvalues, int64_t* out_buckets, uint64_t* out_counts, uint64_t cap_groups,
                         uint8_t* out_key_bytes, uint64_t cap_key_bytes, uint64_t* out_key_offsets, uint64_t* out_entry_offsets,
                         uint16_t* out_entry_ranges, uint64_t* out_entry_hits, uint64_t cap_entries, uint64_t out_info[6]);
/* The vmrange index of one number (Histogram.Update above), -1 for a number it skips: host build of the mapping the kernel runs.  For tests. */
int vlscan_vmrange_index(double v);
/* The vmrange text of index 0 .. VLSCAN_VMRANGES - 1 (%.3e ends, initBucketRanges): its length (no NUL written), -1 when cap is too small, -2 for
 * an index out of range. */
int vlscan_vmrange_text(uint32_t index, char* buf, size_t cap);
/* ---- the N newest selected rows: `/select/logsql/query?limit=N` (app/vlselect/logsql/logsql.go:932-948, 1005-1080 getLastNQueryResults) ---------
 * Same preconditions as the gather calls: the result of the last vlscan_scan_resident of the ctx, whose batch must still be alive.  Every block
 * with selected rows must have been staged with its timestamps.  The call leaves that result as it was: vlscan_fetch_results, the gather calls
 * and vlscan_hits_stats return afterwards what they returned before it.
 *   rows: the selected rows with _time >= min_timestamp, ordered by (timestamp, block index, row); the last min(limit, count) of them are
 *     returned in that ascending order (getLastNRows after sortLogRows; among equal timestamps the later rows win, across blocks the higher
 *     block index, so the result is deterministic).  A caller that merges batches passes the N-th newest timestamp it holds so far as
 *     min_timestamp: the batch then returns only rows that can still enter the merged result (INTEGRATION.md §3d).
 *   field_names: canonical names ("" = _msg); "_time" is rejected (it is out_timestamps).  The text of field f of returned row i is exactly what
 *     vlscan_gather_values yields for that row: out_bytes[out_offsets[i * nfields + f], out_offsets[i * nfields + f + 1]) (out_offsets has
 *     cap_rows * nfields + 1 entries).
 * Output per row: out_timestamps[i], out_blocks[i] (block index in the batch), out_rows[i] (row in its block).
 * out_info (may be NULL) = {rows returned, value bytes, selected rows, blocks whose timestamps were decoded}; it is filled also when the call fails
 * because cap_rows or cap_bytes is too small (then nothing else is written).  Blocks are pruned by their headers: only blocks whose maximum
 * timestamp reaches the weighted limit-th largest block minimum are looked at row by row, and blocks whose minimum equals their maximum are
 * never decoded.  A block whose decoded timestamps contradict its header fails the call.  At most 2^32 - 2 selected rows per batch. */
typedef struct vlscan_last_query {
    uint64_t limit;                /* N >= 1                                                                                       */
    int64_t min_timestamp;         /* rows older than this are not candidates (INT64_MIN = no floor)                               */
    uint32_t nfields;              /* fields to return for each row                                                                */
    const char* const* field_names;
    const size_t* field_name_lens;
} vlscan_last_query;
int vlscan_last_rows(vlscan_ctx* ctx, const vlscan_last_query* q, int64_t* out_timestamps, uint32_t* out_blocks, uint32_t* out_rows, uint64_t cap_rows,
                     uint8_t* out_bytes, uint64_t cap_bytes, uint64_t* out_offsets, uint64_t out_info[4]);
/* ---- facets: `| facets N max_values_per_field M max_value_len L` over the selected rows (/select/logsql/facets, app/vlselect/logsql/logsql.go:31-106) ----
 * The state one pipeFacetsProcessorShard (lib/logstorage/pipe_facets.go:162-307) holds after it saw the selected rows of the last vlscan_scan_resident
 * of the ctx; limit, the skip of const fields and the merge of batches stay with the caller (INTEGRATION.md §3e).  Same preconditions as the gather
 * calls; the call leaves the scan result as it was.  Blocks with selected rows must have been staged with timestamps when `_time` is a field.
 *   field_names: canonical names ("" = _msg), "_time" for the timestamps; at least one, no duplicates, no `_stream` / `_stream_id` (streams are
 *     unknown to the engine).  A field a block does not have adds nothing for that block.
 *   what a block adds to a field (updateFacetsForColumn): a const value with the block's selected rows as hits; each dict entry with selected rows;
 *     every selected row's uint8..uint64 / int64 number; and the text of every other value as vlscan_gather_values yields it (`_time`: RFC3339Nano,
 *     UTC).  Texts skip "" and are keyed like hitsMapAdaptive.updateStateGeneric: a text tryParseUint64 accepts is that number ("1_000" and a uint16
 *     1000 are one entry), a '-' text tryParseInt64 accepts is a negative-class number ("-0" is not the uint64 0), anything else is its bytes.
 *   dropped: a field with a value longer than max_value_len (numbers by uint64StringLen / int64StringLen when max_value_len <= 20 / 21), or with
 *     more than max_values_per_field distinct entries.  Its state is only that flag.  A table of the next power of two >= 2 * min(max_values_per_field
 *     + 1, selected rows) slots per field lives on the device; a max_values_per_field whose tables do not fit fails the call.
 * Output: out_dropped[f] (0 kept, 1 dropped); the entries of field f are [out_field_offsets[f], out_field_offsets[f + 1]) (nfields + 1 offsets),
 * ordered by hits descending, then text bytewise, then class (VLSCAN_FACET_UINT64 < _NEGATIVE < _STRING); entry e has out_hits[e], out_classes[e] and
 * the text out_bytes[out_value_offsets[e], out_value_offsets[e + 1]) (marshalUint64String / marshalInt64String for the two number classes).
 * out_info (may be NULL) = {entries, value bytes, selected rows, blocks whose timestamps were decoded}; it is filled also when the call fails because
 * cap_entries or cap_bytes is too small (then nothing else is written).  `_time` decodes only blocks whose minimum differs from their maximum.
 * At most 2^32 - 2 selected rows per batch. */
enum { VLSCAN_FACET_UINT64 = 0, VLSCAN_FACET_NEGATIVE = 1, VLSCAN_FACET_STRING = 2 };
#define VLSCAN_FACETS_DEFAULT_MAX_VALUES 1000    /* pipeFacetsDefaultMaxValuesPerField */
#define VLSCAN_FACETS_DEFAULT_MAX_VALUE_LEN 128  /* pipeFacetsDefaultMaxValueLen */
typedef struct vlscan_facets_query {
    uint64_t max_values_per_field;   /* 0 = VLSCAN_FACETS_DEFAULT_MAX_VALUES                                                       */
    uint64_t max_value_len;          /* 0 = VLSCAN_FACETS_DEFAULT_MAX_VALUE_LEN                                                    */
    uint32_t nfields;
    const char* const* field_names;
    const size_t* field_name_lens;
} vlscan_facets_query;
int vlscan_facets(vlscan_ctx* ctx, const vlscan_facets_query* q, uint8_t* out_dropped, uint64_t* out_field_offsets, uint64_t* out_hits, uint8_t* out_classes,
                  uint64_t cap_entries, uint8_t* out_bytes, uint64_t cap_bytes, uint64_t* out_value_offsets, uint64_t out_info[4]);
/* Digest of the last scan's bitmaps of the blocks [block_lo, block_hi) of its batch, computed on the device: xor over the blocks of
 * XXH64(the block's bitmap words as little-endian bytes) * (2 * (key_base + block index) + 1).  The oracle reports the same quantity for its own
 * bitmaps, so a bench can check a billion-row scan against the CPU restatement on any block range without moving the bitmaps.  The batch of the
 * last scan must still be alive (like for vlscan_fetch_hits: both read its block table on the device). */
int vlscan_result_digest(vlscan_ctx* ctx, uint64_t block_lo, uint64_t block_hi, uint64_t key_base, uint64_t* out_digest);
/* Multi-GPU hosts (one process, several devices): blocks are independent, so the Go side gives every GPU its own vlscan_ctx
 * (vlscan_ctx_create(worker_id % vlscan_device_count())) and its own share of the block list; nothing is exchanged on the data path.  The only
 * reduction of a query like `| stats count()` is this sum of the four match counters {rows, rows_matched, blocks_matched, values_bytes} of the
 * last scan of every ctx (it synchronises each ctx's stream).  Multi-process jobs (bench.py: one rank per GPU) reduce the same vector with
 * one NCCL all-reduce instead (vlscan_result_device_ptrs gives its device address). */
int vlscan_totals_sum(vlscan_ctx* const* ctxs, int nctx, uint64_t out4[4]);
/* Device pointers of the last scan's results (bench / multi-GPU reduce): bitmap words, per-block counts,
 * and a 4 x u64 totals vector {rows, rows_matched, blocks_matched, values_bytes}. */
int vlscan_result_device_ptrs(vlscan_ctx* ctx, void** bitmap_words, void** match_counts, void** totals4);

/* End-to-end call on host buffers: upload + scan + fetch + free (what the cgo shim calls per work batch; replaces the body of the worker loop,
 * storage_search.go:1044-1062).  Only what the program can read crosses PCIe:
 *  - bloom filters of fields no leaf / no AND-OR pre-pass ever probes stay on the host;
 *  - when the program does probe bloom filters the call is staged bloom-first, in the reference's lazy order (getBloomFilterForColumn
 *    block_search.go:411-439 before getValuesForColumn :444-474): headers + bloom filters, a probe pass on the device, then only the values of
 *    the (block, column) cells some filter can reach (vlscan_stats.staged_columns / pruned_columns).  Results and accounting are identical to
 *    staging in one go.  $VLSCAN_BLOOM_FIRST: 0 = never, 2 = always, 1 (default) = adaptive (skipped for 7 calls after a probe that left
 *    less than 1/8 of the values bytes on the host);
 *  - VLSCAN_STAGE_ONDISK payloads travel compressed and are regenerated in HBM.  Page-locked inputs go out as a few large DMA transfers;
 *    pageable ones (a part's mmap()ed files) are packed through a pinned ring by $VLSCAN_HOST_THREADS threads of the ctx, launch group by
 *    launch group, while the device decodes the previous group.
 * The batch object is recycled inside the ctx; nothing of the call outlives it except out_bitmap_words / out_match_counts / stats. */
int vlscan_scan_batch(vlscan_ctx* ctx, const vlscan_program* prog, const char* const* field_names, const size_t* field_name_lens,
                      uint32_t nfields, const vlscan_block* blocks, uint64_t nblocks, uint64_t* out_bitmap_words,
                      uint32_t* out_match_counts, vlscan_stats* stats);
/* ---- keeping an end-to-end scan on the device: the pipes' columns staged only for the blocks that need them (DESIGN.md §3.12) -----------------
 * The reference reads the columns the pipes need only after the filter left a non-empty bitmap (block_search.go:217-225).
 * vlscan_scan_batch_keep: vlscan_scan_batch with the same arguments, bitmaps, counts and counters, whose batch stays the ctx's last result: the
 *   gather calls, vlscan_fetch_*, vlscan_result_digest, vlscan_hits_stats, vlscan_last_rows and vlscan_facets work on it until the next
 *   vlscan_scan_resident, vlscan_scan_batch or vlscan_scan_batch_keep on the ctx, or vlscan_ctx_free.  The device memory is the ctx's and is reused
 *   by the next call.  The field list may name fields the program does not reference (output fields).  Staging is always split into headers and
 *   values: const values and dict tables of every field go with the headers; the values of the program's fields are staged for the blocks the
 *   bloom probe lets through (when the program probes and VLSCAN_BLOOM_FIRST lets it, as in vlscan_scan_batch) or for every block; the values of
 *   output fields stay on the host.  Timestamps are staged for every block that has them.  The counters are vlscan_scan_batch's except for
 *   h2d_bytes, gpu_launches and the timings: staged_columns / pruned_columns are filled when the bloom probe ran, 0 / 0 otherwise.  An empty
 *   field list or an empty batch is accepted as by vlscan_scan_batch.
 * vlscan_stage_selected: stages the values of the named fields of the kept batch for the listed blocks (block_list, nlist entries) or, with
 *   block_list == NULL, for every block with selected rows.  `blocks` / `nblocks` must be the descriptors the keep call was given (the library
 *   never retains caller pointers): block count, and for the blocks read, rows, column count, and per column field, kind, value type, stage
 *   and payload lengths (on-disk: the values bytes; decoded: lens items and data, each) are checked against what that call saw (<0 on a mismatch).  Cells already staged, const cells and absent fields are
 *   skipped; a field the kept batch was not staged with is an error, and so is an empty field list (a caller with nothing to stage skips the
 *   call).  May be called several times; what it stages lives as long as the kept
 *   batch.  out_info (filled on success) = {cells staged, cells skipped because already staged, host->device bytes, bytes blocks (ZSTD or
 *   plain) run through the device decoder}.
 * A gather, vlscan_hits_stats, vlscan_last_rows or vlscan_facets that needs the values of a cell still on the host fails with an error naming
 * the field; the ctx and the kept result stay usable.  A failure of vlscan_stage_selected while it stages ends the kept result. */
int vlscan_scan_batch_keep(vlscan_ctx* ctx, const vlscan_program* prog, const char* const* field_names, const size_t* field_name_lens,
                           uint32_t nfields, const vlscan_block* blocks, uint64_t nblocks, uint64_t* out_bitmap_words,
                           uint32_t* out_match_counts, vlscan_stats* stats);
int vlscan_stage_selected(vlscan_ctx* ctx, const vlscan_block* blocks, uint64_t nblocks, const char* const* field_names, const size_t* field_name_lens,
                          uint32_t nfields, const uint32_t* block_list /* NULL = every block with selected rows */, uint64_t nlist, uint64_t out_info[4]);

#ifdef __cplusplus
}
#endif
#endif /* VLSCAN_H */
