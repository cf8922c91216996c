/*
 * lz4b200.h — C ABI of the H100-native (sm_90a) LZ4 block codec (liblz4b200.so).
 *
 * This is the drop-in boundary for lz4_flex's block path.  lz4_flex has no FFI of its own:
 * its boundary is the crate's public Rust API.  Every entry point below names the Rust item
 * (file:line in the lz4_flex v0.12.0 source tree) whose work it takes over; INTEGRATION.md shows the
 * `extern "C"` block + safe wrappers a maintainer adds on the Rust side.
 *
 * Conventions
 *   - plain pointers and sizes only; the caller owns every buffer; the library never hands
 *     out memory the caller must free (ownership rule of SURVEY.md §8b).
 *   - every function returns an lz4b200_status; bad *data* is never a crash, always a code
 *     (mirrors Result<_, DecompressError/CompressError>, src/block/mod.rs:82-106).
 *   - "device" variants take device pointers and a CUDA stream (cudaStream_t passed as
 *     void*; NULL is the legacy default stream, lz4b200_ctx_stream() the context's own),
 *     enqueue work and return without synchronising.  Launches of one context must be
 *     stream-ordered with respect to each other (they share the context's ticket counters
 *     and scratch).  "host" variants take host
 *     pointers, stage through pinned memory and return when the result is in the caller's
 *     buffer.
 *   - all functions are thread-safe for distinct contexts; one context may be used by one
 *     thread at a time (FrameEncoder/FrameDecoder are &mut self in the reference, too).
 */
#ifndef LZ4B200_H
#define LZ4B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LZ4B200_ABI_VERSION 1

/* Status codes.  1..6 are the reference's error enums:
 *   CompressError::OutputTooSmall                    src/block/mod.rs:103-106
 *   DecompressError::{OutputTooSmall{expected,actual}, LiteralOutOfBounds,
 *                     ExpectedAnotherByte, OffsetZero, OffsetOutOfBounds}   src/block/mod.rs:82-98
 * 101..115 are frame::Error variants (src/frame/mod.rs:35-72). */
typedef enum lz4b200_status {
    LZ4B200_OK = 0,
    LZ4B200_COMPRESS_OUTPUT_TOO_SMALL = 1,
    LZ4B200_DEC_OUTPUT_TOO_SMALL = 2,
    LZ4B200_DEC_LITERAL_OUT_OF_BOUNDS = 3,
    LZ4B200_DEC_EXPECTED_ANOTHER_BYTE = 4,
    LZ4B200_DEC_OFFSET_ZERO = 5,
    LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS = 6,

    LZ4B200_FRAME_DECOMPRESSION_ERROR = 101, /* Error::DecompressionError(block code)   */
    LZ4B200_FRAME_WRONG_MAGIC = 102,         /* Error::WrongMagicNumber                 */
    LZ4B200_FRAME_RESERVED_BITS = 103,       /* Error::ReservedBitsSet                  */
    LZ4B200_FRAME_UNSUPPORTED_VERSION = 104, /* Error::UnsupportedVersion               */
    LZ4B200_FRAME_UNSUPPORTED_BLOCKSIZE = 105,/* Error::UnsupportedBlocksize            */
    LZ4B200_FRAME_HEADER_CHECKSUM = 106,     /* Error::HeaderChecksumError              */
    LZ4B200_FRAME_BLOCK_CHECKSUM = 107,      /* Error::BlockChecksumError               */
    LZ4B200_FRAME_CONTENT_CHECKSUM = 108,    /* Error::ContentChecksumError             */
    LZ4B200_FRAME_CONTENT_LENGTH = 109,      /* Error::ContentLengthError               */
    LZ4B200_FRAME_BLOCK_TOO_BIG = 110,       /* Error::BlockTooBig                      */
    LZ4B200_FRAME_SKIPPABLE = 111,           /* Error::SkippableFrame                   */
    LZ4B200_FRAME_DICTIONARY = 112,          /* Error::DictionaryNotSupported           */
    LZ4B200_FRAME_IO_EOF = 113,              /* Error::IoError(UnexpectedEof)           */
    LZ4B200_FRAME_LINKED_UNSUPPORTED = 114,  /* BlockMode::Linked asked of the ENCODER (the decoder handles it) */
    LZ4B200_FRAME_OUTPUT_FULL = 115,         /* caller's flat output buffer exhausted   */

    LZ4B200_INVALID_ARGUMENT = 200,
    LZ4B200_CUDA_ERROR = 201
} lz4b200_status;

/* How a block is parsed by the encoder (SURVEY.md §8a "Modes").  Bit 0: CONT — the block is
 * compressed as FrameEncoder compresses every block but the first of a table epoch: stream
 * offset > 0, so position 0 is not pre-inserted and empty slots never match
 * (src/frame/compress.rs:357-367, src/block/compress.rs:353-359,403-429).
 * Bit 1: HASH5_ALWAYS — use the 5-byte hash + u32-table rule even below 65 535 bytes, as
 * FrameEncoder does (src/frame/compress.rs:77,140; src/block/hashtable.rs:41-44).
 * The block API (compress_into & co) uses 0 for every block. */
#define LZ4B200_BLOCK_FRESH         0u
#define LZ4B200_BLOCK_CONT          1u
#define LZ4B200_BLOCK_HASH5_ALWAYS  2u

typedef struct lz4b200_ctx lz4b200_ctx;

/* ---- library / context --------------------------------------------------------------- */

int lz4b200_abi_version(void);
/* How this library's CUDA runtime sees a host pointer: 0 pageable, 1 pinned, 2 device, 3 managed, -1 unknown.
 * The host batch calls overlap PCIe traffic with kernels only for pinned (page-locked) buffers. */
int lz4b200_host_pointer_kind(const void *p);
const char *lz4b200_status_string(int status);
/* Last CUDA error text seen by this context (empty string if none). */
const char *lz4b200_last_cuda_error(const lz4b200_ctx *ctx);

/* One context per (thread, GPU): owns a stream, pinned staging and device scratch.
 * Fails with LZ4B200_CUDA_ERROR when no usable device exists — there is no CPU fallback. */
lz4b200_status lz4b200_ctx_create(int device, lz4b200_ctx **out);
void lz4b200_ctx_destroy(lz4b200_ctx *ctx);
/* Ask for the highest CUDA stream priority for this context's host-batch pipelines (call before the first
 * batch call).  Use it for the decompress side when a compress context keeps the same GPU busy: decode kernels are
 * short and otherwise queue behind the encoder's long-lived CTAs. */
void lz4b200_ctx_set_priority(lz4b200_ctx *ctx, int high);
/* The context's own stream (cudaStream_t). */
void *lz4b200_ctx_stream(lz4b200_ctx *ctx);
/* Name of the kernel the launcher picked for the context's last compress (which = 0) / decompress (which = 1) batch —
 * diagnostics only: bench.py records it beside the roofline so a profile is never attributed to the wrong kernel.  The name
 * carries the template arguments of the instantiation that ran.  A compress batch whose `max_in_len` exceeds 64 KiB
 * names the encoder of blocks above 64 KiB; one with `max_in_len` 0, or whose dictionary takes dict_len + max_in_len
 * above 64 KiB, runs that encoder as well as the one of the smaller blocks and names both, joined by " + ". */
const char *lz4b200_ctx_last_kernel(const lz4b200_ctx *ctx, int which);

/* ---- sizes ------------------------------------------------------------------------------ */

/* block::get_maximum_output_size — src/block/compress.rs:588-590. */
size_t lz4b200_max_output_size(size_t input_len);

/* ---- block API, one block, host pointers -------------------------------------------------
 * 1:1 replacements.  One call = one block = ONE serial parse chain on the GPU: a 64 KiB block costs milliseconds to
 * compress and decompress however empty the machine is (a CPU core needs tens of microseconds) — these calls are
 * chain-latency-bound, not PCIe-bound.  They exist for drop-in completeness; throughput comes from the batch calls,
 * which run thousands of such chains at once (INTEGRATION.md section 2, "Which call"). */

/* block::compress_into — src/block/compress.rs:599-601.  Fails up-front with
 * COMPRESS_OUTPUT_TOO_SMALL when cap < lz4b200_max_output_size(n) (compress.rs:338-340). */
lz4b200_status lz4b200_compress_into(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                     uint8_t *out, size_t cap, size_t *written);

/* block::compress_prepend_size — src/block/compress.rs:673-675 (u32 LE length + block). */
lz4b200_status lz4b200_compress_prepend_size(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                             uint8_t *out, size_t cap, size_t *written);

/* block::decompress_into — src/block/decompress.rs:454-456.  On DEC_OUTPUT_TOO_SMALL,
 * *err_expected / *err_actual carry the enum's fields (decompress.rs:350-354,403-406). */
lz4b200_status lz4b200_decompress_into(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                       uint8_t *out, size_t cap, size_t *written,
                                       size_t *err_expected, size_t *err_actual);

/* block::decompress_size_prepended — src/block/decompress.rs:496-499 with
 * block::uncompressed_size — src/block/mod.rs:151-157.  `cap` must be >= the prefixed size
 * (query it with lz4b200_uncompressed_size first); decoding uses exactly the prefixed size
 * as capacity like the reference's Vec::with_capacity. */
lz4b200_status lz4b200_uncompressed_size(const uint8_t *in, size_t n, size_t *size);
lz4b200_status lz4b200_decompress_size_prepended(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                 uint8_t *out, size_t cap, size_t *written,
                                                 size_t *err_expected, size_t *err_actual);

/* ---- block API, many independent blocks, DEVICE pointers (the measured hot path) ----------
 * Block b reads  d_in  + in_off[b]  (in_len[b] bytes)
 *       writes   d_out + out_off[b] (at most out_cap[b] bytes; out_len[b] = bytes produced)
 * All descriptor arrays live in device memory.  Work is enqueued on `stream`.  A context carries the
 * work-distribution counters (and the encoder's global hash tables) of ONE batch call at a time: calls on the same
 * context must be stream-ordered; use one context per concurrently running stream or host thread.
 * Per-block results: d_status[b] (lz4b200_status) and, for decode, d_err_expected[b]
 * (the `expected` of OutputTooSmall; `actual` is out_cap[b]).  A failed block never disturbs
 * its neighbours. */

/* compress_internal over many blocks — src/block/compress.rs:318-489.  d_flags may be NULL
 * (all blocks LZ4B200_BLOCK_FRESH = block API semantics).  Each out_cap[b] must be >=
 * lz4b200_max_output_size(in_len[b]) or the block reports COMPRESS_OUTPUT_TOO_SMALL.
 * `max_in_len` is a host-known upper bound of in_len[] (0 = unknown): blocks of up to 64 KiB
 * and larger blocks run in differently-shaped kernels, and the bound lets the launcher skip
 * the one with no work. */
lz4b200_status lz4b200_compress_batch_device(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len,
    const uint8_t *d_flags,
    uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap,
    uint32_t *d_out_len, int32_t *d_status, size_t nblocks,
    uint32_t max_in_len, void *stream);

/* decompress_internal over many blocks — src/block/decompress.rs:201-449. */
lz4b200_status lz4b200_decompress_batch_device(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len,
    uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap,
    uint32_t *d_out_len, int32_t *d_status, uint64_t *d_err_expected,
    size_t nblocks, void *stream);

/* ---- block API, many independent blocks, HOST pointers (end-to-end path) ------------------
 * Host arrays; includes H2D of inputs and D2H of results (pinned host memory gives full
 * PCIe speed, pageable memory works).  Compressed blocks come back PACKED: block b is
 * written at out + out_off[b] where out_off[] is an OUTPUT (out_off[b+1] = out_off[b] +
 * out_len[b]), so only the produced bytes cross PCIe; `out_cap_total` bounds the sum.
 * Decompress: bytes of an output slot past the block's decoded length are overwritten with zeros (the reference
 * leaves them unspecified: wild copies, SURVEY.md §8a); nothing of an earlier call can appear there. */
lz4b200_status lz4b200_compress_batch_host(lz4b200_ctx *ctx,
    const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len, const uint8_t *flags,
    uint8_t *out, size_t out_cap_total, uint64_t *out_off,
    uint32_t *out_len, int32_t *status, size_t nblocks);

lz4b200_status lz4b200_decompress_batch_host(lz4b200_ctx *ctx,
    const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
    uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
    uint32_t *out_len, int32_t *status, uint64_t *err_expected, size_t nblocks);

/* block::compress_into_with_table — src/block/compress.rs:744-766, CompressTable :709-735.  The reusable table
 * only selects the table layout / hash of the parse: LZ4B200_TABLE_SMALL = u16 entries + 4-byte hash (inputs
 * < 65 535 bytes), LZ4B200_TABLE_LARGE = u32 entries + 5-byte hash (any size).  A SMALL table given an input of
 * >= 65 535 bytes is upgraded to LARGE and stays LARGE (compress.rs:750-752): *table_kind is that in/out state. */
#define LZ4B200_TABLE_SMALL 0
#define LZ4B200_TABLE_LARGE 1
lz4b200_status lz4b200_compress_into_with_table(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                uint8_t *out, size_t cap, size_t *written, int *table_kind);

/* ---- external dictionary ("_with_dict") -----------------------------------------------------
 * The dictionary logically precedes the input: the encoder may reference its last 64 KiB, the decoder
 * resolves offsets that reach before the start of the output inside it.  Like the reference, the
 * encoder ignores dictionaries of <= 3 bytes (compress.rs:626-628) and everything but the last
 * WINDOW_SIZE = 65 536 bytes (init_dict, compress.rs:571-575); the table layout / hash follow
 * dict_len + n (compress.rs:559).  One dictionary is shared by every block of a batch. */

/* block::compress_into_with_dict — src/block/compress.rs:610-616 (compress_with_dict :685-687). */
lz4b200_status lz4b200_compress_into_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                               const uint8_t *dict, size_t dict_len,
                                               uint8_t *out, size_t cap, size_t *written);

/* block::compress_prepend_size_with_dict — src/block/compress.rs:692-694. */
lz4b200_status lz4b200_compress_prepend_size_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                       const uint8_t *dict, size_t dict_len,
                                                       uint8_t *out, size_t cap, size_t *written);

/* block::decompress_into_with_dict — src/block/decompress.rs:462-468 (copy_from_dict :85-109;
 * DEC_OFFSET_OUT_OF_BOUNDS when offset > bytes written + dict_len, :287-289/:399-401). */
lz4b200_status lz4b200_decompress_into_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                 const uint8_t *dict, size_t dict_len,
                                                 uint8_t *out, size_t cap, size_t *written,
                                                 size_t *err_expected, size_t *err_actual);

/* block::decompress_size_prepended_with_dict — src/block/decompress.rs:522-528. */
lz4b200_status lz4b200_decompress_size_prepended_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                           const uint8_t *dict, size_t dict_len,
                                                           uint8_t *out, size_t cap, size_t *written,
                                                           size_t *err_expected, size_t *err_actual);

/* Batches with one shared dictionary: device pointers (d_dict on the device) and host pointers. */
lz4b200_status lz4b200_compress_batch_device_with_dict(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len,
    const uint8_t *d_dict, size_t dict_len,
    uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap,
    uint32_t *d_out_len, int32_t *d_status, size_t nblocks,
    uint32_t max_in_len, void *stream);
lz4b200_status lz4b200_decompress_batch_device_with_dict(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len,
    const uint8_t *d_dict, size_t dict_len,
    uint8_t *d_out, const uint64_t *d_out_off, const uint32_t *d_out_cap,
    uint32_t *d_out_len, int32_t *d_status, uint64_t *d_err_expected,
    size_t nblocks, void *stream);
lz4b200_status lz4b200_compress_batch_host_with_dict(lz4b200_ctx *ctx,
    const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
    const uint8_t *dict, size_t dict_len,
    uint8_t *out, size_t out_cap_total, uint64_t *out_off,
    uint32_t *out_len, int32_t *status, size_t nblocks);
lz4b200_status lz4b200_decompress_batch_host_with_dict(lz4b200_ctx *ctx,
    const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
    const uint8_t *dict, size_t dict_len,
    uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
    uint32_t *out_len, int32_t *status, uint64_t *err_expected, size_t nblocks);

/* ---- many size-prepended blocks, DEVICE pointers ----------------------------------------------------------------------
 * A record is what block::compress_prepend_size writes: the input's length as a u32 LE word, then its block
 * (src/block/compress.rs:673-675, src/block/mod.rs:151-157).  Every array lives in device memory.  Argument errors return
 * INVALID_ARGUMENT before anything is enqueued, every output untouched: a null ctx or d_rec_off / d_out_off; with a
 * non-empty batch a null input, descriptor or per-record array, or a null d_out with out_cap > 0; a count above
 * UINT32_MAX; a null dictionary with dict_len > 0.  An empty batch writes 0 to d_rec_off[0] / d_out_off[0] and nothing
 * else.  Otherwise the work is enqueued on `stream` and the call returns without synchronising (a call larger than any
 * before it on the context first grows the context's scratch, and CUDA may synchronise while it frees and allocates).
 * Like every device call, calls on one context must be ordered on one stream: they share the context's ticket counters
 * and scratch.  d_in, d_out and the dictionary may have any alignment; d_out's bytes past the last written record are
 * not written. */

/* block::compress_prepend_size — src/block/compress.rs:673-675 — for each of many blocks, the records packed back to
 * back.  Block b is d_in[in_off[b], in_off[b] + in_len[b]), compressed as the block API does (every block FRESH).
 * Record b is exactly the bytes lz4b200_compress_prepend_size writes for that input; d_rec_off[b] is its offset in
 * d_out and d_rec_off[nblocks] the total the batch needs (d_rec_off has nblocks + 1 entries).
 * d_status[b]: OK, or COMPRESS_OUTPUT_TOO_SMALL when
 *   - in_len[b] > max_in_len: max_in_len is a host bound on every in_len; it sizes the scratch, one slot of
 *     lz4b200_max_output_size(max_in_len) per block, and such a block's slot is too small.  Its record takes 0 bytes.
 *   - the record does not fit: d_rec_off[b] + its length > out_cap.  Nothing of it is written, but its length counts in
 *     d_rec_off, so d_rec_off[nblocks] is what to allocate.
 * The kernel that compresses the blocks is the one lz4b200_compress_batch_device picks for the same batch and
 * max_in_len. */
lz4b200_status lz4b200_compress_prepend_size_batch_device(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, size_t nblocks, uint32_t max_in_len,
    uint8_t *d_out, size_t out_cap, uint64_t *d_rec_off, int32_t *d_status, void *stream);

/* block::compress_prepend_size_with_dict — src/block/compress.rs:692-694 — the same with one dictionary shared by every
 * block, normalised as lz4b200_compress_batch_device_with_dict does (ignored at <= 3 bytes, the last 64 KiB kept):
 * record b is the bytes of lz4b200_compress_prepend_size_with_dict. */
lz4b200_status lz4b200_compress_prepend_size_batch_device_with_dict(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_in_off, const uint32_t *d_in_len, size_t nblocks, uint32_t max_in_len,
    const uint8_t *d_dict, size_t dict_len,
    uint8_t *d_out, size_t out_cap, uint64_t *d_rec_off, int32_t *d_status, void *stream);

/* block::decompress_size_prepended — src/block/decompress.rs:496-499 — for each of many records, with no host
 * synchronisation: the length words set the output layout on the device.  Record b is d_in[rec_off[b], rec_off[b] +
 * rec_len[b]).  d_out_off[b] is the sum of the length words of records 0..b-1 (a record of fewer than 4 bytes counts 0)
 * and d_out_off[nrec] the total (d_out_off has nrec + 1 entries).  Record b decodes into d_out + d_out_off[b] with a
 * capacity of exactly its length word, the reference's Vec::with_capacity.  d_status[b], d_out_len[b] and
 * d_err_expected[b] (may be NULL) are the status, *written and *err_expected lz4b200_decompress_size_prepended returns
 * for those bytes (err_actual is the length word), and the decoded bytes are the same:
 *   - fewer than 4 bytes: DEC_EXPECTED_ANOTHER_BYTE (src/block/mod.rs:152);
 *   - a region that ends past out_cap: INVALID_ARGUMENT (the one-record call's cap < size rule); nothing is written.
 * Bytes of a region past d_out_len[b] are what lz4b200_decompress_batch_device leaves there: a decoded record leaves
 * them untouched, a record that fails may leave there bytes it decoded before the error.  They are not zeroed (the host
 * calls zero them).  The kernel that decodes is the one lz4b200_decompress_batch_device picks for nrec blocks. */
lz4b200_status lz4b200_decompress_size_prepended_batch_device(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_rec_off, const uint32_t *d_rec_len, size_t nrec,
    uint8_t *d_out, size_t out_cap, uint64_t *d_out_off, uint32_t *d_out_len,
    int32_t *d_status, uint64_t *d_err_expected, void *stream);

/* block::decompress_size_prepended_with_dict — src/block/decompress.rs:522-528 — the same with one dictionary shared by
 * every record (the last 64 KiB kept, as lz4b200_decompress_batch_device_with_dict does). */
lz4b200_status lz4b200_decompress_size_prepended_batch_device_with_dict(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_rec_off, const uint32_t *d_rec_len, size_t nrec,
    const uint8_t *d_dict, size_t dict_len,
    uint8_t *d_out, size_t out_cap, uint64_t *d_out_off, uint32_t *d_out_len,
    int32_t *d_status, uint64_t *d_err_expected, void *stream);

/* ---- frame format (encoder: independent blocks; decoder: independent and linked) -------------
 * FrameInfo — src/frame/header.rs:130-192. */
typedef struct lz4b200_frame_info {
    int32_t block_size_id;     /* BlockSize: 0 Auto, 4 64KB, 5 256KB, 6 1MB, 7 4MB (header.rs:39-53) */
    int32_t block_checksums;   /* FrameInfo::block_checksums   */
    int32_t content_checksum;  /* FrameInfo::content_checksum  */
    int32_t has_content_size;  /* FrameInfo::content_size.is_some() */
    uint64_t content_size;     /* FrameInfo::content_size      */
    int32_t linked;            /* BlockMode::Linked — the encoder rejects it (LZ4B200_FRAME_LINKED_UNSUPPORTED) */
    int32_t reserved;
} lz4b200_frame_info;

/* Upper bound of the frame produced from n input bytes with this FrameInfo. */
size_t lz4b200_frame_bound(size_t n, const lz4b200_frame_info *info);

/* FrameEncoder::with_frame_info(info, w); w.write_all(in); finish()
 *   — src/frame/compress.rs:128-187,234-404.  `first_write_len` is the length of the first
 * write() call (it only matters for BlockSize::Auto, header.rs:57-67); pass n for a single
 * write_all.  Host pointers. */
lz4b200_status lz4b200_frame_compress(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                      const lz4b200_frame_info *info, size_t first_write_len,
                                      uint8_t *out, size_t cap, size_t *written);

/* FrameEncoder::with_frame_info(info, w); w.write_all(in); finish() — src/frame/compress.rs:128-187,234-404 — for input in
 * DEVICE memory, written to DEVICE memory.  For every input, info and first_write_len it returns the status
 * lz4b200_frame_compress returns, and d_out[0, *d_written) holds the bytes that call writes.  Argument errors are
 * reported before anything is enqueued.  Otherwise the work is enqueued on `stream` and the call returns without
 * synchronising; *d_written (a device u64) receives the frame length.  d_in and d_out may have any alignment; bytes of
 * d_out past the frame are not written. */
lz4b200_status lz4b200_frame_compress_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n,
                                             const lz4b200_frame_info *info, size_t first_write_len,
                                             uint8_t *d_out, size_t cap, uint64_t *d_written, void *stream);

/* FrameEncoder::with_frame_info(info_f, w); w.write_all(in_f); finish() for each of many inputs in DEVICE memory, written
 * back to back into DEVICE memory in one call.  Input f is d_in[in_off[f], in_off[f] + in_len[f]); in_off and in_len are
 * HOST arrays of nframes entries, d_frame_off a DEVICE array of nframes + 1.  info_f is *info with two changes: block
 * size Auto (0) resolves from in_len[f] (an Auto batch mixes block sizes), and with has_content_size set frame f's
 * header records in_len[f] (info->content_size is ignored).  d_out[d_frame_off[f], d_frame_off[f + 1]) holds exactly
 * the bytes lz4b200_frame_compress(ctx, host copy of input f, in_len[f], &info_f, in_len[f], ...) writes; frames lie
 * back to back from d_out[0], d_frame_off[nframes] is the total, and nothing of d_out past it is written.
 * Argument errors, reported before anything is enqueued (d_out and d_frame_off untouched), in this order:
 *   INVALID_ARGUMENT           a null ctx, info or d_frame_off; a null in_off, in_len or d_out with nframes > 0; a null
 *                              d_in with a non-empty input;
 *   FRAME_LINKED_UNSUPPORTED   linked blocks;
 *   INVALID_ARGUMENT           a block size id other than 0 or 4..7; nframes or the batch's block count above UINT32_MAX;
 *   COMPRESS_OUTPUT_TOO_SMALL  out_cap < the sum of lz4b200_frame_bound(in_len[f], &info_f).
 * nframes == 0 sets d_frame_off[0] = 0.  Otherwise all planning is done on the host, the work is enqueued on `stream`
 * and the call returns without synchronising; calls on one context must be ordered on one stream, as for every device
 * call.  d_in and d_out may have any alignment and must not overlap.  Device scratch is one slot of
 * lz4b200_max_output_size(block length) per block, about the size of the input; there is no budget. */
lz4b200_status lz4b200_frame_compress_batch_device(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *in_off, const uint64_t *in_len,
    const lz4b200_frame_info *info,
    uint8_t *d_out, size_t out_cap, uint64_t *d_frame_off,
    size_t nframes, void *stream);

/* Block-range form used for multi-GPU sharding (SURVEY.md §8e): compress frame blocks
 * [first_block, first_block + nblocks) of a stream cut into `block_size`-byte blocks.  `d_in`
 * points at the first byte of block `first_block` (device memory, `in_len` bytes for this
 * range); block k's mode is derived from its absolute index exactly like
 * FrameEncoder::write_block (frame/compress.rs:266-271,357-367).  Output: for each block a
 * 4-byte BlockInfo followed by the payload (raw copy when compression does not shrink it,
 * frame/compress.rs:301-306), written back-to-back into d_out in block order;
 * *d_total = bytes written.  d_block_sizes[k] = 4 + payload bytes (may be NULL).
 * Everything stays on the device; enqueued on `stream`. */
lz4b200_status lz4b200_frame_compress_blocks_device(lz4b200_ctx *ctx,
    const uint8_t *d_in, size_t in_len, size_t block_size, uint64_t first_block,
    uint8_t *d_out, size_t out_cap, uint64_t *d_total, uint32_t *d_block_sizes, void *stream);

/* The same work in two steps, for the sharded (multi-GPU) frame path of SURVEY.md §8e: _range_compress leaves the
 * range's compressed / stored blocks in the context and writes the packed size to *d_total (device); _range_pack lays
 * the [BlockInfo | payload] segments out at d_dst + *d_dst_offset (device scalar; NULL = 0).  d_dst may be PEER
 * memory — rank 0's frame buffer mapped with lz4b200_peer_open — so the pack kernel's stores are the NVLink transfer of
 * the gather step (frame/compress.rs:261-371 writes the same bytes to its io::Write in block order). */
lz4b200_status lz4b200_frame_range_compress(lz4b200_ctx *ctx, const uint8_t *d_in, size_t in_len, size_t block_size,
                                            uint64_t first_block, uint64_t *d_total, uint32_t *d_block_sizes,
                                            void *stream);
lz4b200_status lz4b200_frame_range_pack(lz4b200_ctx *ctx, uint8_t *d_dst, const uint64_t *d_dst_offset, void *stream);

/* Buffers shared between the ranks of one node (CUDA IPC, one process per GPU): the owner allocates and gets a
 * 64-byte handle to pass around (any transport); the others map it and may hand the mapping to _range_pack. */
lz4b200_status lz4b200_peer_alloc(lz4b200_ctx *ctx, size_t bytes, void **d_ptr, uint8_t *handle64);
lz4b200_status lz4b200_peer_open(lz4b200_ctx *ctx, const uint8_t *handle64, void **d_ptr);
lz4b200_status lz4b200_peer_close(lz4b200_ctx *ctx, void *d_ptr);
lz4b200_status lz4b200_peer_free(lz4b200_ctx *ctx, void *d_ptr);

/* Bytes of scratch-free output space the call above needs in the worst case. */
size_t lz4b200_frame_blocks_bound(size_t in_len, size_t block_size);

/* Writes the frame header for `info` (7..15 bytes) — FrameInfo::write, header.rs:232-275. */
size_t lz4b200_frame_write_header(const lz4b200_frame_info *info, uint8_t *out, size_t cap);

/* ONE frame: FrameDecoder::new(r).read_to_end() — src/frame/decompress.rs:109-342, 352-422.  The reference's
 * reader returns Ok(0) at every EndMark (decompress.rs:310-331; tests/tests.rs:633-647 reads two concatenated frames
 * with two read_to_end calls), so the unit of this call is the frame that starts at in[0]: it is decoded into `out`,
 * *consumed receives the input bytes it occupied (header, blocks, EndMark, content checksum) and the caller calls
 * again with in + *consumed for the next frame.  n == 0, or 4 bytes of magic followed by the end of the input
 * (decompress.rs:113-128), is a clean end: OK with *written == 0.
 *   - bytes decoded before a corrupt block / truncation are delivered (*written) together with the error;
 *   - *block_status receives the block decoder's code for FRAME_DECOMPRESSION_ERROR; *err_expected / *err_actual
 *     receive ContentLengthError{expected, actual} (frame/mod.rs) or the block's OutputTooSmall{expected, actual}.
 *     OutputTooSmall is relative to the failing block on every frame path, linked frames included: expected = the
 *     bytes the block had decoded + the literal run or match that did not fit, actual = the block size.  Two ways the
 *     reference differs on linked frames, neither replicated: its decoder writes after the frame's earlier output in
 *     one buffer, so its expected and actual also count that prefix (frame/decompress.rs:196-305); and once
 *     that buffer has wrapped (an ext_dict window), a block decodes into the buffer's head and can pass the block
 *     size without an error.  Here a block that decodes to more than the block size is always DEC_OUTPUT_TOO_SMALL;
 *   - frames with linked blocks (frame/decompress.rs:196-222, 277-305; what `lz4`, LZ4F and pyarrow write by
 *     default) are decoded too: their blocks form a dependency chain that the device resolves in stream order;
 *   - device memory is bounded: independent blocks are decoded in groups whose output slots
 *     (min(block size, 255 x payload) each) fit lz4b200_ctx_set_frame_budget() bytes (default 256 MiB), reusing the
 *     slots from group to group — the reference decodes any frame in O(block size) memory.
 * lz4b200_ctx_set_frame_budget (at least 1 MiB) bounds the device memory of the frame decoders and of the streaming
 * frame encoder (lz4b200_frame_encoder, below): per group, the decoders' slots and staged input, and the encoder's
 * buffered input and slots. */
lz4b200_status lz4b200_frame_decompress_next(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                             uint8_t *out, size_t cap, size_t *consumed, size_t *written,
                                             int *block_status, uint64_t *err_expected, uint64_t *err_actual);
void lz4b200_ctx_set_frame_budget(lz4b200_ctx *ctx, size_t bytes);

/* Convenience: every concatenated frame of `in` through lz4b200_frame_decompress_next, outputs back to back
 * (stops at the first error; frame boundaries are not reported — use _next when they matter). */
lz4b200_status lz4b200_frame_decompress(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                        uint8_t *out, size_t cap, size_t *written,
                                        int *block_status);

/* Upper bound of the decoded size of all frames in `in`: per block min(frame block size, 255 x payload) (stored
 * blocks: their length).  The header's content_size is deliberately ignored (untrusted).  Host-side walk only. */
lz4b200_status lz4b200_frame_decoded_bound(const uint8_t *in, size_t n, size_t *bound);

/* lz4b200_frame_decompress_next for ONE frame whose bytes are in DEVICE memory, decoded into DEVICE memory.  For every
 * input and every `cap` it returns what lz4b200_frame_decompress_next returns for the same bytes in host memory: status,
 * consumed, written, block_status, err_expected, err_actual and the first `written` bytes of d_out (bytes of d_out past
 * `written` are not written).  The header, the BlockInfo chain, the block checksums and the content checksum are
 * processed on the GPU; only block descriptors (16 B per block) and per-group statuses cross PCIe.  d_in may have any
 * alignment.  Work is enqueued on `stream` (NULL = legacy default stream, lz4b200_ctx_stream() = the context's own); the
 * call synchronises that stream and returns with the result in d_out.  The result scalars are host pointers. */
lz4b200_status lz4b200_frame_decompress_next_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n, uint8_t *d_out,
                                                    size_t cap, size_t *consumed, size_t *written, int *block_status,
                                                    uint64_t *err_expected, uint64_t *err_actual, void *stream);

/* lz4b200_frame_decoded_bound for frames in device memory (every concatenated frame; content_size ignored); the walk runs
 * on the GPU on `stream`, which the call synchronises. */
lz4b200_status lz4b200_frame_decoded_bound_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n, size_t *bound,
                                                  void *stream);

/* What lz4b200_frame_decompress_next returns for one frame: its status and its five result scalars. */
typedef struct lz4b200_frame_result {
    uint64_t consumed, written, err_expected, err_actual;
    int32_t status, block_status;
} lz4b200_frame_result;                          /* 40 bytes */

/* Many independent frames in DEVICE memory, decoded into DEVICE memory in one call.  Frame f is the frame that starts
 * at d_in + d_frame_off[f], in a region of d_frame_len[f] bytes; d_results[f] receives exactly what
 * lz4b200_frame_decompress_next returns on the same context (same frame budget) for those bytes in host memory with
 * cap = d_out_cap[f], and d_out[d_out_off[f], +written) the bytes it writes.  Nothing else of d_out is written.  A
 * region that holds several concatenated frames decodes only the first (`consumed` says where it ended).  Output
 * regions must not overlap (not checked).  Every array is in device memory.  INVALID_ARGUMENT, before anything is
 * enqueued: a null ctx, a null array with nframes > 0, nframes > UINT32_MAX; nframes == 0 does nothing.  A frame's own
 * error goes into its result and does not affect any other frame.  The frames' blocks are decoded together, many
 * frames per launch; the call synchronises `stream` before it returns. */
lz4b200_status lz4b200_frame_decompress_batch_device(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_frame_off, const uint64_t *d_frame_len,
    uint8_t *d_out, const uint64_t *d_out_off, const uint64_t *d_out_cap,
    lz4b200_frame_result *d_results, size_t nframes, void *stream);

/* ---- random access into one frame in DEVICE memory (no lz4_flex counterpart) ------------------------------------------
 * A frame records no decoded block sizes, so reading content bytes [a, b) of a frame means decoding it from its first
 * block.  lz4b200_frame_index_device builds, on the GPU, the decoded offset and length of every block without decoding
 * it; lz4b200_frame_decompress_ranges_device then decodes only the blocks that many byte ranges touch. */
typedef struct lz4b200_frame_index_entry {
    uint64_t payload_off;         /* the block's payload, from the frame's first byte */
    uint64_t decoded_off;         /* the block's first content byte */
    uint32_t word;                /* the BlockInfo word: payload length | 0x80000000 for a stored block */
    uint32_t decoded_len;         /* the block's decoded bytes */
} lz4b200_frame_index_entry;      /* 24 bytes */

typedef struct lz4b200_frame_index_info {
    uint64_t block_size;          /* the frame's maximum block size in bytes (8 MiB for legacy frames) */
    uint64_t nblocks;             /* entries the index holds: the blocks before the first failing block */
    uint64_t content_len;         /* their decoded total */
    int32_t linked;               /* BlockMode::Linked */
    int32_t pad;
    lz4b200_frame_result result;  /* the frame's result, as lz4b200_frame_decompress_next_device returns it */
} lz4b200_frame_index_info;       /* 72 bytes */

/* Indexes the frame that starts at d_in[0] (the unit of lz4b200_frame_decompress_next_device).  The header and the
 * BlockInfo chain are walked on the GPU, block checksums are verified there when the frame has them, and one GPU thread
 * per block walks its token stream, reading only the compressed bytes: it makes every check the block decoder makes, in
 * the same order, so a block it accepts decodes without error.  A device prefix sum then gives the decoded offsets.
 *   - with d_index NULL the call only walks the chain and writes the blocks it records to *nblocks: a count to allocate
 *     by.  Otherwise *nblocks receives the entries the call needs, the blocks before the first that fails its checksum;
 *     with max_blocks below that the call returns INVALID_ARGUMENT having written only *nblocks.
 *   - d_index[0, info->nblocks) receive the entries; entries past info->nblocks up to *nblocks may be written.
 *   - info->result equals, field by field, what lz4b200_frame_decompress_next_device returns for the same bytes with a
 *     sufficient cap, except that the content checksum is never verified (that needs every decoded byte): where that
 *     call returns FRAME_CONTENT_CHECKSUM the index reports OK.  FRAME_CONTENT_LENGTH is reported.  info->content_len is
 *     the device call's `written`: the decoded total of the indexed blocks.
 *   - a linked frame's offsets that reach before a block are valid when they stay within the frame's earlier output;
 *     the walk records how far each block reaches back and the check runs once the decoded offsets are known.
 * The returned status is the call's own (INVALID_ARGUMENT, CUDA_ERROR) or OK; the frame's status is info->result.status.
 * Work runs on `stream`, which the call synchronises; info and nblocks are host pointers, d_index device memory.
 * The context's scratch holds a descriptor and the sizing results of every block while the call runs. */
lz4b200_status lz4b200_frame_index_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n,
                                          lz4b200_frame_index_entry *d_index, size_t max_blocks, size_t *nblocks,
                                          lz4b200_frame_index_info *info, void *stream);

/* Decodes content bytes [d_start[i], d_start[i] + d_len[i]) of the indexed frame at d_in[0, n) into
 * d_out + d_out_off[i], for i < nranges, in one call.  Ranges are clipped to info->content_len like a Python slice, and
 * d_written[i] receives the clipped length.  Nothing else of d_out is written; ranges may overlap each other in the
 * frame, their outputs must not overlap (not checked).  Every array is in device memory; info is a host pointer.
 *   - independent blocks: the blocks a range touches are found on the device by binary search over the decoded offsets.
 *     A compressed block that lies wholly inside a range decodes straight into d_out; a range's partial first and last
 *     blocks decode into context scratch and are copied out; stored blocks are copied.  Work goes in windows of blocks
 *     whose scratch fits the frame budget (at least one block); ranges in chunks of 65 536.
 *   - linked blocks: the touched blocks form segments of consecutive blocks, each with a look-back of the blocks that
 *     hold the 64 KiB of content before it.  A segment's blocks decode in parallel without their window: each output
 *     byte is its value or a marker naming the earlier byte it copies.  Markers then resolve in block order.  A segment
 *     with a requested byte that copies content before its look-back decodes again with the look-back doubled (in
 *     blocks), up to block 0; segments whose look-backs meet merge.  On English text (dickens, 64 KiB blocks) the
 *     look-back stays 2-4 blocks; on data that copies itself from block to block (a file tiled over and over, such as
 *     repeated JSON or logs) it reaches block 0.  Entries take four bytes per content byte, in windows that fit the
 *     frame budget (at least one block and 64 KiB of carry).
 *   - the index is untrusted: its info and every entry are checked against n, the block size and each other before
 *     anything is decoded (INVALID_ARGUMENT), and every decoded block must produce exactly its indexed length
 *     (FRAME_DECOMPRESSION_ERROR; d_out's range regions then hold unspecified bytes).  Block checksums are not verified
 *     again.
 * INVALID_ARGUMENT before anything is enqueued: a null ctx or info, a null array with nranges > 0, a null d_in with
 * n > 0, a null d_index with info->nblocks > 0.  Work runs on `stream`, which the call synchronises. */
lz4b200_status lz4b200_frame_decompress_ranges_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n,
                                                      const lz4b200_frame_index_info *info,
                                                      const lz4b200_frame_index_entry *d_index,
                                                      const uint64_t *d_start, const uint64_t *d_len, uint8_t *d_out,
                                                      const uint64_t *d_out_off, uint64_t *d_written, size_t nranges,
                                                      void *stream);

/* Block decodes the context's last lz4b200_frame_decompress_ranges_device call ran: for a linked frame every block of
 * every round, look-back included; for independent blocks the (range, block) items.  0 after a call that decoded
 * nothing.  A diagnostic: it shows how far random access into a frame reached back. */
uint64_t lz4b200_ctx_last_range_blocks(const lz4b200_ctx *ctx);

/* d_bound[f] = what lz4b200_frame_decoded_bound gives for region f when it holds one frame (the first frame's bound
 * when it holds several).  Enqueued on `stream`; the call returns without synchronising.  Argument errors as above. */
lz4b200_status lz4b200_frame_decoded_bound_batch_device(lz4b200_ctx *ctx,
    const uint8_t *d_in, const uint64_t *d_frame_off, const uint64_t *d_frame_len,
    uint64_t *d_bound, size_t nframes, void *stream);

/* Streaming frame decoder over DEVICE memory: FrameDecoder (frame/decompress.rs:109-342), which reads a frame one
 * block at a time, for compressed bytes that arrive in HBM chunk by chunk (a GPUDirect Storage reader, a network
 * receive) and decoded output taken in caller-sized pieces.  Its device memory does not depend on the frame's length:
 * the context's frame budget (slots and staged payload), the caller's buffers, and the decoder's own 128 KiB (a linked
 * frame's 64 KiB window, double-buffered) and hash state.  Linked frames (what `lz4`, LZ4F and pyarrow write by
 * default) cross calls and groups through the window.  Linked decoding is still one serial chain per frame.
 * A decoder belongs to one context; destroy it before the context.  Its persistent state (walk position, header
 * fields, output so far, window, content hash) is its own; descriptors, slots and staged payload are the context's
 * scratch, so other calls on the context, another decoder's included, may run between two of its calls, ordered on
 * one stream as every device call of a context is. */
typedef struct lz4b200_frame_decoder lz4b200_frame_decoder;
lz4b200_status lz4b200_frame_decoder_create(lz4b200_ctx *ctx, lz4b200_frame_decoder **out);
void lz4b200_frame_decoder_destroy(lz4b200_frame_decoder *dec);

typedef struct lz4b200_frame_decoder_step {
    uint64_t consumed;            /* bytes of d_in this call used: whole units only */
    uint64_t written;             /* d_out[0, written) was written; nothing past it */
    uint64_t need;                /* stopped for lack of input: at least this many bytes from d_in + consumed make the
                                     next unit; else 0 */
    int32_t frame_done;           /* 1: the frame ended in this call, and `result` is its result */
    int32_t pad;
    lz4b200_frame_result result;  /* the frame's result as lz4b200_frame_decompress_next returns it (below) */
} lz4b200_frame_decoder_step;     /* 72 bytes */

/* Continues the frame in progress with d_in[0, n), or starts one at d_in[0]; decodes into d_out[0, out_cap).
 *   - input: a call takes whole units only (the header; a block: BlockInfo, payload and block checksum; the EndMark
 *     with the content checksum).  The caller presents the unconsumed rest again, with more bytes after it.  With
 *     end_of_input == 0, running out of input is never an error: the call stops and sets `need`.  With end_of_input
 *     set, d_in runs to the end of the input, and a truncated unit ends the frame as _next reports it.
 *   - output: the call decodes consecutive whole blocks while the sum of their decoded bounds (min(block size,
 *     255 x payload); a stored block its length) fits out_cap, and while the group loop would not cut them (their slots
 *     and input span fit the frame budget).  At most 65 536 blocks per call: a call may stop with need == 0 and input
 *     left, and the caller calls again.  When the next block's bound alone exceeds out_cap the call returns
 *     LZ4B200_FRAME_OUTPUT_FULL having consumed nothing, and the decoder is as it was.  An out_cap of at least the
 *     frame's block size (8 MiB for legacy frames) always makes progress.
 *   - frames: a call never crosses a frame boundary.  When the frame ends (EndMark, an error, or the end of input),
 *     frame_done = 1 and the next call starts a new frame, as the reference's reader returns Ok(0) at each EndMark.
 *     At end_of_input with nothing left the result is _next's for empty input: OK, 0 consumed, 0 written.
 *   - the result: over every chunking of a frame F (end_of_input on the last chunk) and every out_cap of at least
 *     its block size, the concatenated `written` bytes are what lz4b200_frame_decompress_next(F, cap = decoded bound)
 *     writes, and `result` holds its status, written (the frame's total), block_status, err_expected, err_actual and
 *     consumed (the frame's total).  One exception: after a block decode error (FRAME_DECOMPRESSION_ERROR) _next's
 *     consumed is where its whole-frame walk ended, while the decoder's is the end of the failing block and its
 *     checksum, where the reference's reader stands at that point.  Errors keep stream order: a decode error in an
 *     earlier block wins over a later block's checksum failure, which cuts the frame at that block.
 *   - INVALID_ARGUMENT, before anything is enqueued: a null decoder or step, a null d_in with n > 0, a null d_out with
 *     out_cap > 0.  d_in and d_out may have any alignment.  Work runs on `stream`, which the call synchronises before
 *     it returns; `step` is host memory. */
lz4b200_status lz4b200_frame_decoder_decode_device(lz4b200_frame_decoder *dec, const uint8_t *d_in, size_t n,
                                                   int end_of_input, uint8_t *d_out, size_t out_cap,
                                                   lz4b200_frame_decoder_step *step, void *stream);

/* Streaming frame encoder over DEVICE memory: FrameEncoder (frame/compress.rs:62-404), an io::Write over any number of
 * write_all, flush and try_finish calls, for input that a GPU producer writes in pieces (a checkpoint writer, a
 * GPUDirect Storage writer, a simulation dumping fields) or that is too large to be resident at once.  Its device
 * memory does not depend on the stream's length or on a call's length: one input buffer of a group of whole blocks,
 * the context's slots and descriptors for that group, and about 14 KiB of its own (hash state and output position).
 * A group is as many blocks as fit the context's frame budget (lz4b200_ctx_set_frame_budget), each counting its block
 * size of buffer and its lz4b200_max_output_size(block size) slot; at least one block.  At the default 256 MiB budget a
 * group of 64 KiB blocks is 1 950 blocks.  The buffer is (re)allocated when a frame opens, the point where BlockSize
 * Auto resolves, and only when the block size or the budget has changed; a frame keeps its group to its end.
 * An encoder belongs to one context; destroy it before the context.  Its state is its own; descriptors and slots are
 * the context's scratch, so other calls on the context, another encoder's or a decoder's included, may run between two
 * of its calls, ordered on one stream as every device call of a context is.
 * create: INVALID_ARGUMENT for a null ctx, info or out, or a block size id other than 0 or 4..7;
 * FRAME_LINKED_UNSUPPORTED for linked blocks. */
typedef struct lz4b200_frame_encoder lz4b200_frame_encoder;
lz4b200_status lz4b200_frame_encoder_create(lz4b200_ctx *ctx, const lz4b200_frame_info *info,
                                            lz4b200_frame_encoder **out);
void lz4b200_frame_encoder_destroy(lz4b200_frame_encoder *enc);

#define LZ4B200_ENCODE_WRITE  0   /* write_all(d_in)                 */
#define LZ4B200_ENCODE_FLUSH  1   /* write_all(d_in); flush()        */
#define LZ4B200_ENCODE_FINISH 2   /* write_all(d_in); try_finish()   */

/* The most bytes lz4b200_frame_encoder_encode_device(enc, ., n, op, ...) can write in the encoder's current state: the
 * header when the call opens a frame, 4 + length (+ 4 with block checksums) for every block of every group the call
 * completes, and for FINISH the EndMark (+ 4 with a content checksum).  0 for a null encoder or an unknown op. */
size_t lz4b200_frame_encoder_bound(const lz4b200_frame_encoder *enc, size_t n, int op);

/* content_len of the open (or last) frame: the input bytes it has taken so far.  With a FRAME_CONTENT_LENGTH result it
 * is the `actual` of ContentLengthError{expected, actual}. */
uint64_t lz4b200_frame_encoder_content_len(const lz4b200_frame_encoder *enc);

/* write_all(d_in[0, n)), then flush() (FLUSH) or try_finish() (FINISH), writing the call's bytes to d_out[0, *d_written).
 *   - output: over any sequence of calls on one encoder (empty writes, flushes, finishes, writes after a finish, which
 *     open the next frame), the concatenated d_out[0, *d_written) of the calls are what lz4_flex's FrameEncoder writes
 *     for the same sequence of write_all / flush / try_finish, quirks included: Auto resolves from the first non-empty
 *     write of the first frame and stays resolved for later frames; FINISH with nothing written writes an empty frame
 *     (header and EndMark); a second FINISH writes a second EndMark (and the last frame's digest); the stream state is
 *     reset when a frame opens after a frame that had content.  Only when the bytes appear differs: input is buffered
 *     and compressed in whole groups.  Bytes of d_out past *d_written are not written.
 *   - buffering: the input is copied into the encoder's buffer; each time it holds a full group, the group is
 *     compressed and the buffer empties.  FLUSH and FINISH compress what is buffered, the last block short.  The caller
 *     may reuse d_in once `stream` has passed the call.  Each block's parse mode follows the stream offset
 *     (compress.rs:266-271, 357-367), planned on the host; after a flush it is not the block index's.
 *   - the groups of a call pack back to back after the header, which is written only when the call opens a frame.  Block
 *     checksums are computed one GPU thread per block; the content hash runs over each group's input in stream order and
 *     is finished by the kernel that writes the EndMark.
 *   - errors, reported before anything is enqueued, the encoder, d_out and *d_written untouched, in this order:
 *       INVALID_ARGUMENT           a null encoder or d_written, a null d_out with out_cap > 0; a null d_in with n > 0;
 *                                  an op other than LZ4B200_ENCODE_WRITE, _FLUSH or _FINISH;
 *       COMPRESS_OUTPUT_TOO_SMALL  out_cap < lz4b200_frame_encoder_bound(enc, n, op).
 *   - FINISH when the frame records a content size other than its content_len behaves as try_finish does
 *     (compress.rs:209-219): the flushed blocks are written and counted in *d_written, no EndMark is written, the frame
 *     is closed and the call returns FRAME_CONTENT_LENGTH.
 *   - the work is enqueued on `stream` and the call returns without synchronising; *d_written is a device u64.  Only
 *     kernel arguments and each group's parse modes cross PCIe.  d_in and d_out may have any alignment and must not
 *     overlap. */
lz4b200_status lz4b200_frame_encoder_encode_device(lz4b200_frame_encoder *enc, const uint8_t *d_in, size_t n, int op,
                                                   uint8_t *d_out, size_t out_cap, uint64_t *d_written, void *stream);

/* Device bytes the context holds now, its scratch included (a diagnostic). */
size_t lz4b200_ctx_device_bytes(const lz4b200_ctx *ctx);

/* XXH32 (twox-hash XxHash32, Cargo.toml:51) — used for header/block/content checksums.
 * The streaming form backs FrameEncoder's running content hash (frame/compress.rs:141,320). */
uint32_t lz4b200_xxh32(const uint8_t *data, size_t n, uint32_t seed);
typedef struct lz4b200_xxh32_state {
    uint32_t acc[4];
    uint8_t buf[16];
    uint32_t fill;
    uint32_t seed;
    uint64_t total;
} lz4b200_xxh32_state;
void lz4b200_xxh32_reset(lz4b200_xxh32_state *st, uint32_t seed);
void lz4b200_xxh32_update(lz4b200_xxh32_state *st, const uint8_t *data, size_t n);
uint32_t lz4b200_xxh32_digest(const lz4b200_xxh32_state *st);

#ifdef __cplusplus
}
#endif
#endif /* LZ4B200_H */
