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
 * diagnostics only: bench.py records it beside the roofline so a profile is never attributed to the wrong kernel. */
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
 *     receive ContentLengthError{expected, actual} (frame/mod.rs) or the block's OutputTooSmall{expected, actual};
 *   - frames with linked blocks (frame/decompress.rs:196-222, 277-305; what `lz4`, LZ4F and pyarrow write by
 *     default) are decoded too: their blocks form a dependency chain that the device resolves in stream order;
 *   - device memory is bounded: independent blocks are decoded in groups whose output slots
 *     (min(block size, 255 x payload) each) fit lz4b200_ctx_set_frame_budget() bytes (default 256 MiB), reusing the
 *     slots from group to group — the reference decodes any frame in O(block size) memory. */
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
