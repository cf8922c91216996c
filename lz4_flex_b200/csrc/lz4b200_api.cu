// lz4b200_api.cu — host runtime and C ABI (include/lz4b200.h) of the H100 (sm_90a) LZ4 block codec.
//
// Everything here is product code: contexts, launch plumbing, host<->device staging and the
// frame container (header / BlockInfo / checksums), which is host-side bookkeeping around the
// two block kernels.  There is no CPU codec in this library: without a CUDA device every entry
// point that has work to do fails with LZ4B200_CUDA_ERROR.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "lz4b200_frame_batch.cuh"
#include "lz4b200_frame_encoder.cuh"
#include "lz4b200_frame_range.cuh"
#include "lz4b200_frame_walk.cuh"
#include "lz4b200_kernels.cuh"
#include "lz4b200_solo_kernel.cuh"
#ifdef LZ4B200_AB_VARIANTS
// A/B build (lz4_flex_b200/liblz4b200_ab.so, -DLZ4B200_AB_VARIANTS): the kernels that lost their measurements stay
// compilable and testable there (tests/test_gpu_kernel_variants.py) but are not part of the product library.
#include "lz4b200_thread_kernels.cuh"
#endif

using namespace lz4b200;

// ---------------------------------------------------------------------------------------------
// small device helpers used by the frame path
// ---------------------------------------------------------------------------------------------
namespace lz4b200 {

// Exclusive scan of sizes[0..n) into offs[0..n], offs[n] = total.  One CTA; n is a block count
// (<= a few 100k), so a single-CTA chunked scan is far below launch noise.
__global__ void __launch_bounds__(1024) scan_sizes_kernel(const uint32_t *sizes, uint64_t *offs, uint32_t n)
{
    __shared__ uint64_t warp_sums[32];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        uint32_t i = base + threadIdx.x;
        uint64_t v = i < n ? sizes[i] : 0, x = v;
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t y = __shfl_up_sync(kFull, x, d);
            if ((threadIdx.x & 31) >= d) x += y;
        }
        if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint64_t w = warp_sums[threadIdx.x], s = w;
            for (int d = 1; d < 32; d <<= 1) {
                uint64_t y = __shfl_up_sync(kFull, s, d);
                if (threadIdx.x >= d) s += y;
            }
            warp_sums[threadIdx.x] = s - w;
        }
        __syncthreads();
        uint64_t excl = carry + warp_sums[threadIdx.x >> 5] + x - v;
        if (i < n) offs[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) offs[n] = carry;
}

// Generic gather: segment b copies len[b] bytes from src_base[sel] + src_off[b] to dst + dst_off[b],
// optionally preceded by a 4-byte little-endian word (the frame BlockInfo).  One CTA per segment
// slice; byte-granular head/tail, 16-byte body when co-aligned.
struct GatherArgs {
    const uint8_t *src_a;          // segment source when pick[b] == 0
    const uint8_t *src_b;          // segment source when pick[b] != 0
    const uint64_t *off_a;
    const uint64_t *off_b;
    const uint32_t *len_a;
    const uint32_t *len_b;
    const uint8_t *pick;           // may be null (always a)
    const uint32_t *prefix_word;   // may be null; else written as 4 LE bytes before the payload
    uint8_t *dst;
    const uint64_t *dst_off;
    uint32_t nseg;
    const uint64_t *dst_shift = nullptr;   // optional device scalar added to every destination offset
};

__global__ void __launch_bounds__(256) gather_segments_kernel(GatherArgs g)
{
    for (uint32_t b = blockIdx.x; b < g.nseg; b += gridDim.x) {
        const bool second = g.pick && g.pick[b];
        const uint8_t *s = second ? g.src_b + g.off_b[b] : g.src_a + g.off_a[b];
        const uint32_t len = second ? g.len_b[b] : g.len_a[b];
        uint8_t *d = g.dst + g.dst_off[b] + (g.dst_shift ? *g.dst_shift : 0ull);
        if (g.prefix_word) {
            if (threadIdx.x < 4) d[threadIdx.x] = (uint8_t)(g.prefix_word[b] >> (8 * threadIdx.x));
            d += 4;
        }
        const uint32_t dm = (uint32_t)(reinterpret_cast<uintptr_t>(d) & 15u);
        const uint32_t sm = (uint32_t)(reinterpret_cast<uintptr_t>(s) & 15u);
        if (dm == sm && len >= 64) {
            uint32_t head = (16u - dm) & 15u;
            if (threadIdx.x < head) d[threadIdx.x] = s[threadIdx.x];
            uint32_t body = (len - head) >> 4;
            const uint4 *s4 = reinterpret_cast<const uint4 *>(s + head);
            uint4 *d4 = reinterpret_cast<uint4 *>(d + head);
            for (uint32_t i = threadIdx.x; i < body; i += blockDim.x) d4[i] = s4[i];
            uint32_t done = head + (body << 4);
            if (done + threadIdx.x < len) d[done + threadIdx.x] = s[done + threadIdx.x];
        } else {
            for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) d[i] = s[i];
        }
    }
}

// Frame encoder bookkeeping for a block range: per block, decide compressed-vs-stored
// (frame/compress.rs:301-306) and produce BlockInfo word + segment size.  `trailer` (0, or 4 for a
// block checksum) is reserved after each payload.
__global__ void frame_block_info_kernel(const uint32_t *comp_len, const uint32_t *raw_len, uint32_t n, uint32_t trailer,
                                        uint32_t *info_word, uint8_t *pick_raw, uint32_t *seg_size,
                                        uint32_t *payload_len)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t c = comp_len[i], r = raw_len[i];
    bool stored = !(c < r);
    info_word[i] = stored ? (r | 0x80000000u) : c;
    pick_raw[i] = stored ? 1 : 0;
    payload_len[i] = stored ? r : c;
    seg_size[i] = 4u + (stored ? r : c) + trailer;
}

// Descriptor generator for a run of equal-sized blocks cut from one contiguous buffer.
__global__ void make_uniform_desc_kernel(uint64_t total_len, uint32_t block, uint64_t out_stride,
                                         uint64_t first_block, uint64_t fresh_period, uint32_t n,
                                         uint64_t *in_off, uint32_t *in_len, uint64_t *out_off,
                                         uint32_t *out_cap, uint8_t *flags)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t o = (uint64_t)i * block;
    uint64_t rem = total_len - o;
    in_off[i] = o;
    in_len[i] = (uint32_t)(rem < block ? rem : block);
    out_off[i] = (uint64_t)i * out_stride;
    out_cap[i] = (uint32_t)out_stride;
    uint64_t k = first_block + i;
    bool fresh = (k % fresh_period) == 0;
    flags[i] = (uint8_t)(LZ4B200_BLOCK_HASH5_ALWAYS | (fresh ? 0u : LZ4B200_BLOCK_CONT));
}

// ---- many size-prepended blocks (lz4b200_compress_prepend_size_batch_device & co) ---------------------------------------
// A record is the input's length as a u32 LE word followed by its block (compress.rs:673-675, block/mod.rs:151-157).

// The compressor's arguments, one thread per block: block b's slot is b x `slot` bytes.  A block longer than max_in_len
// goes in empty with no room, which every encoder reports as COMPRESS_OUTPUT_TOO_SMALL (given its real length, the
// encoder of small blocks would skip it and leave its status unwritten when max_in_len keeps the other one from running).
__global__ void __launch_bounds__(128) prepend_desc_kernel(const uint32_t *in_len, uint32_t n, uint32_t max_in_len,
                                                           uint32_t slot, uint32_t *len, uint64_t *out_off, uint32_t *out_cap)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    const bool fits = in_len[b] <= max_in_len;
    len[b] = fits ? in_len[b] : 0u;
    out_off[b] = (uint64_t)b * slot;
    out_cap[b] = fits ? slot : 0u;
}

// Record sizes for the scan: the length word and the block, nothing for a block the encoder refused.
__global__ void __launch_bounds__(128) prepend_size_kernel(const uint32_t *out_len, const int32_t *status, uint32_t n,
                                                           uint32_t *size)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n) size[b] = status[b] == LZ4B200_OK ? 4u + out_len[b] : 0u;
}

// A record that ends past out_cap fails and is not written.  The others get their length word here and their block from
// the gather (dst, glen); the gather's own prefix word is written unconditionally, so it cannot skip a record.
__global__ void __launch_bounds__(128) prepend_place_kernel(const uint32_t *in_len, const uint32_t *out_len,
                                                            const uint64_t *rec_off, uint32_t n, uint64_t out_cap,
                                                            uint8_t *out, int32_t *status, uint64_t *dst, uint32_t *glen)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    const uint64_t o = rec_off[b];
    bool live = status[b] == LZ4B200_OK;
    if (live && o + 4u + out_len[b] > out_cap) {
        status[b] = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
        live = false;
    }
    dst[b] = o + 4u;
    glen[b] = live ? out_len[b] : 0u;
    if (live)
        for (int i = 0; i < 4; i++) out[o + i] = (uint8_t)(in_len[b] >> (8 * i));
}

// Each record's length word, read a byte at a time (records start anywhere), is its output size; a record of fewer than
// 4 bytes has none and takes no output.
__global__ void __launch_bounds__(128) prepended_size_kernel(const uint8_t *in, const uint64_t *rec_off,
                                                             const uint32_t *rec_len, uint32_t n, uint32_t *size)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    const uint8_t *p = in + rec_off[b];
    size[b] = rec_len[b] < 4u ? 0u
                              : (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// The decoder's arguments: the block after the length word, decoded in place at out_off[b] with exactly the length word as
// capacity (the reference's Vec::with_capacity).  A record of fewer than 4 bytes goes in empty, for which the decoder
// reports DEC_EXPECTED_ANOTHER_BYTE as the one-record call does; so does a record whose region ends past out_cap, which
// is flagged for prepended_status_kernel.
__global__ void __launch_bounds__(128) prepended_args_kernel(const uint64_t *rec_off, const uint32_t *rec_len,
                                                             const uint32_t *size, const uint64_t *out_off, uint32_t n,
                                                             uint64_t out_cap, uint64_t *in_off, uint32_t *in_len,
                                                             uint32_t *cap, uint8_t *misfit)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n) return;
    const uint32_t len = rec_len[b];
    const bool fits = out_off[b] + size[b] <= out_cap, decode = len >= 4u && fits;
    in_off[b] = rec_off[b] + 4u;
    in_len[b] = decode ? len - 4u : 0u;
    cap[b] = decode ? size[b] : 0u;
    misfit[b] = len >= 4u && !fits;
}

// After the decoder: the one-record call's `cap < want` rule for the records flagged above.
__global__ void __launch_bounds__(128) prepended_status_kernel(const uint8_t *misfit, uint32_t n, int32_t *status)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n && misfit[b]) status[b] = LZ4B200_INVALID_ARGUMENT;
}

// ---- device-resident frame decoder (lz4b200_frame_decompress_next_device) ----------------------------------------------

// One thread walks the frame at `in` (fw::frame_walk, the same code the host path runs), resuming from *w and
// recording at most max_blocks descriptors.
__global__ void frame_walk_kernel(const uint8_t *in, uint64_t n, fw::FrameWalk *w, fw::FrameBlockDesc *out, uint32_t max_blocks)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) fw::frame_walk(in, n, *w, out, max_blocks);
}

// The streaming decoder's walk (lz4b200_frame_decoder): one thread runs fw::frame_walk_stream over the presented chunk.
__global__ void frame_walk_stream_kernel(const uint8_t *in, uint64_t n, bool eof, fw::FrameWalk *w, fw::FrameBlockDesc *out,
                                         uint32_t max_blocks, uint64_t *need)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) fw::frame_walk_stream(in, n, eof, *w, out, max_blocks, need);
}

// A linked frame's window after a group: the last min(64 KiB, old_len + n) bytes of old[0, old_len) followed by
// add[0, n) (the group's output), into dst, which overlaps neither.  The bytes come from wherever they lie, across any
// block or group boundary.
constexpr uint32_t kWindowBytes = 65536;
__global__ void __launch_bounds__(256) window_update_kernel(const uint8_t *old, uint32_t old_len, const uint8_t *add,
                                                            uint64_t n, uint8_t *dst)
{
    const uint64_t total = old_len + n;
    const uint32_t keep = (uint32_t)min(total, (uint64_t)kWindowBytes);
    const uint64_t from = total - keep;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < keep; i += gridDim.x * blockDim.x) {
        const uint64_t p = from + i;
        dst[i] = p < old_len ? old[p] : add[p - old_len];
    }
}

// Block checksums of the blocks the last walk launch recorded (frame indices first .. w->nblocks - 1), one thread per
// block running the serial XXH32 over its payload; *bad receives the lowest index that fails.
__global__ void __launch_bounds__(128) block_checksum_kernel(const uint8_t *in, const fw::FrameBlockDesc *desc,
                                                             const fw::FrameWalk *w, uint64_t first, uint32_t *bad)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (!(w->flg & 0x10) || i >= w->nblocks - first) return;
    if (!fw::block_checksum_ok(in, desc[i])) atomicMin(bad, (uint32_t)(first + i));
}

// The content checksum is one XXH32 chain over the whole content (frame/compress.rs:320, frame/decompress.rs:323-331).
// content_hash_kernel carries the state *st over p[0, n) exactly like fw::xxh32_update, a pending partial stripe at
// entry and exit included: the encoder runs it once over its input, the decoder once per group as the group lands.
// XXH32 is four serial chains, one per 4-byte lane of a 16-byte stripe, each three dependent instructions per word
// (multiply-add, rotate, multiply).  Lanes 0-3 of warp 0 each run one chain over words read from shared memory while
// the other warps stage the next chunk into the second buffer.  The pending stripe is completed byte by byte; the rest
// is staged in 16-byte words from the 16-byte aligned-down address, the partial words at either end byte by byte, so p
// may have any alignment and nothing outside p[0, n) is read.
constexpr uint32_t kHashChunk = 16384;                   // input bytes per staged chunk
constexpr uint32_t kHashChunkWords = kHashChunk / 16;    // 16-byte words (= stripes) per chunk

// Stage the words of chunk c that hold stripe bytes: word w covers a[16w, 16w + 16); bytes outside [lo, hi) are not
// read.  A chunk starting `lo` bytes past an aligned address spans one word more than it has stripes.
__device__ __forceinline__ void hash_stage_chunk(uint8_t *dst, const uint8_t *a, uint64_t lo, uint64_t hi, uint64_t c,
                                                 uint32_t t, uint32_t nt)
{
    const uint64_t w0 = c * kHashChunkWords;
    const uint64_t w1 = min(w0 + kHashChunkWords + 1, (hi + 15) / 16);
    for (uint64_t w = w0 + t; w < w1; w += nt) {
        uint8_t *d = dst + 16 * (w - w0);
        const uint64_t b = 16 * w;
        if (b >= lo && b + 16 <= hi) {
            *reinterpret_cast<uint4 *>(d) = *reinterpret_cast<const uint4 *>(a + b);
        } else {
            for (uint32_t i = 0; i < 16; i++)
                if (b + i >= lo && b + i < hi) d[i] = a[b + i];
        }
    }
}

// One lane's chain over `ns` staged stripes whose first byte is at buf[shift]: word = bytes [off, off + 4) of buf,
// assembled from the two aligned words around it.
__device__ __forceinline__ uint32_t hash_chunk_lane(const uint8_t *buf, uint32_t shift, uint32_t lane, uint32_t acc,
                                                    uint32_t ns)
{
    const uint32_t *s32 = reinterpret_cast<const uint32_t *>(buf);
    const uint32_t r = 8 * (shift & 3);
    uint32_t i = (shift >> 2) + lane;
#pragma unroll 8
    for (uint32_t j = 0; j < ns; j++, i += 4) acc = fw::xxh32_round(acc, __funnelshift_r(s32[i], s32[i + 1], r));
    return acc;
}

// The body of content_hash_kernel, run by every thread of a CTA (shared by the per-frame hash of the batch decoder):
// carries *st (global or shared memory) over p[0, n) using the two staging buffers.
__device__ __forceinline__ void content_hash_cta(lz4b200_xxh32_state *st, const uint8_t *p, uint64_t n,
                                                 uint8_t (*stage)[kHashChunk + 16])
{
    const uint32_t fill = st->fill;
    const uint64_t k = fill ? min((uint64_t)(16u - fill), n) : 0;
    __syncthreads();                                              // every thread has read fill before it changes
    if (threadIdx.x == 0 && k) fw::xxh32_update(*st, p, k);     // complete (or extend) the pending stripe
    __syncthreads();
    const bool pending = st->fill != 0;                           // n too short to complete it: nothing else to do
    uint32_t acc = st->acc[threadIdx.x & 3];
    __syncthreads();                                              // every thread has read *st before it is written
    if (pending) return;

    const uint8_t *q = p + k;
    const uint64_t m = n - k, stripes = m >> 4;
    const uint32_t shift = (uint32_t)(reinterpret_cast<uintptr_t>(q) & 15u);
    const uint8_t *a = q - shift;                                 // 16-byte aligned
    const uint64_t lo = shift, hi = shift + 16 * stripes;         // the stripes' bytes, relative to a
    const uint64_t nchunks = (stripes + kHashChunkWords - 1) / kHashChunkWords;
    if (nchunks) hash_stage_chunk(stage[0], a, lo, hi, 0, threadIdx.x, blockDim.x);
    __syncthreads();
    for (uint64_t c = 0; c < nchunks; c++) {
        if (threadIdx.x < 32) {
            if (threadIdx.x < 4)
                acc = hash_chunk_lane(stage[c & 1], shift, threadIdx.x, acc,
                                      (uint32_t)min((uint64_t)kHashChunkWords, stripes - c * kHashChunkWords));
        } else if (c + 1 < nchunks) {
            hash_stage_chunk(stage[(c + 1) & 1], a, lo, hi, c + 1, threadIdx.x - 32, blockDim.x - 32);
        }
        __syncthreads();
    }
    if (threadIdx.x < 4) st->acc[threadIdx.x] = acc;
    if (threadIdx.x == 0) {
        const uint32_t tail = (uint32_t)(m & 15);
        for (uint32_t i = 0; i < tail; i++) st->buf[i] = q[16 * stripes + i];
        st->fill = tail;
        st->total += m;
    }
}

__global__ void __launch_bounds__(256) content_hash_kernel(lz4b200_xxh32_state *st, const uint8_t *p, uint64_t n)
{
    __shared__ __align__(16) uint8_t stage[2][kHashChunk + 16];
    content_hash_cta(st, p, n, stage);
}

// ---- frame encoders -----------------------------------------------------------------------------------------------------

__global__ void xxh32_reset_kernel(lz4b200_xxh32_state *st, uint32_t seed) { fw::xxh32_reset(*st, seed); }

// Block checksums of a packed range (frame/compress.rs:313-316): the XXH32 of each payload as written (compressed or
// stored), stored little-endian in the 4 trailer bytes after it.  One thread per block.
__global__ void __launch_bounds__(128) frame_block_checksum_kernel(uint8_t *dst, const uint64_t *seg_off,
                                                                   const uint32_t *payload_len, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t *payload = dst + seg_off[i] + 4;
    const uint32_t len = payload_len[i];
    const uint32_t h = fw::xxh32(payload, len, 0);
    for (int b = 0; b < 4; b++) payload[len + b] = (uint8_t)(h >> (8 * b));
}

// ---- streaming frame encoder (lz4b200_frame_encoder) --------------------------------------------------------------------
// The groups of one call pack back to back after the header; *pos is where the next byte of the call's output goes.

// The frame header as a kernel argument (FrameInfo::write is at most 15 bytes).
struct FrameHeaderBytes {
    uint8_t b[19];
    uint8_t len;
};

// The header at out[0] when the call opens a frame (hdr.len 0: none), and *pos = hdr.len.
__global__ void encoder_head_kernel(uint8_t *out, FrameHeaderBytes hdr, uint64_t *pos)
{
#pragma unroll
    for (uint32_t i = 0; i < sizeof hdr.b; i++)
        if (i < hdr.len) out[i] = hdr.b[i];
    *pos = hdr.len;
}

// The end of a call: the EndMark at out[*pos] when the call closes the frame (and the content digest when `content` is
// given), and the call's length into *written.
__global__ void encoder_tail_kernel(uint8_t *out, const uint64_t *pos, bool endmark, const lz4b200_xxh32_state *content,
                                    uint64_t *written)
{
    uint64_t o = *pos;
    if (endmark) {
        for (int b = 0; b < 4; b++) out[o + b] = 0;
        o += 4;
        if (content) {
            const uint32_t h = fw::xxh32_digest(*content);
            for (int b = 0; b < 4; b++) out[o + b] = (uint8_t)(h >> (8 * b));
            o += 4;
        }
    }
    *written = o;
}

// ---- the frame encoders' pipeline (compress_frames) ---------------------------------------------------------------------
// Many frames per call, their blocks numbered frame after frame (fb::FramePlan, one entry per frame, planned on the host).

static_assert(sizeof(fb::FramePlan) == 64, "one frame's plan is 64 bytes");

// A single frame's plan reaches the device as a kernel argument rather than a copy.
__global__ void frame_plan_store_kernel(fb::FramePlan *dst, fb::FramePlan p) { *dst = p; }

// The compressor's arguments, one thread per block of the batch (fb::batch_block); dst[b] receives the block's shift
// into the packed output, to which frame_batch_dst_kernel adds the scan of the segment sizes.
__global__ void __launch_bounds__(128) frame_batch_blocks_kernel(const fb::FramePlan *plan, uint32_t nframes, uint32_t nb,
                                                                 uint64_t *in_off, uint32_t *in_len, uint64_t *out_off,
                                                                 uint32_t *out_cap, uint8_t *flags, uint64_t *dst)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const fb::BlockJob j = fb::batch_block(plan, nframes, b);
    in_off[b] = j.in_off;
    in_len[b] = j.in_len;
    out_off[b] = j.out_off;
    out_cap[b] = j.out_cap;
    flags[b] = j.flags;
    dst[b] = j.dst_shift;
}

// With pos_in, the blocks land *pos_in bytes further (a streaming group at its call's position) and thread 0 stores
// their end to *pos_out, another word than the *pos_in every thread reads.
__global__ void __launch_bounds__(128) frame_batch_dst_kernel(const uint64_t *seg_off, uint32_t nb, uint64_t *dst,
                                                              const uint64_t *pos_in, uint64_t *pos_out)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t pos = pos_in ? *pos_in : 0;
    if (b < nb) dst[b] += seg_off[b] + pos;
    if (b == 0 && pos_out) *pos_out = pos + seg_off[nb];
}

// The content hash of every frame (frame/compress.rs:141,320), one CTA per frame over its input, into states[f].
// (As for frame_batch_hash_kernel, the minimum of one CTA per SM keeps ptxas from a register limit that spills.)
__global__ void __launch_bounds__(256, 1) frame_batch_content_kernel(const uint8_t *in, const fb::FramePlan *plan,
                                                                  lz4b200_xxh32_state *states)
{
    __shared__ __align__(16) uint8_t stage[2][kHashChunk + 16];
    const uint32_t f = blockIdx.x;
    if (threadIdx.x == 0) fw::xxh32_reset(states[f], 0);
    __syncthreads();
    content_hash_cta(states + f, in + plan[f].in_off, plan[f].in_len, stage);
}

// Everything of each frame but its blocks, one thread per frame (frame/compress.rs:209-230): the header, the EndMark,
// the content digest when `states` is given, and frame_off[f]; the last frame's thread also writes the total.
__global__ void __launch_bounds__(128) frame_batch_tail_kernel(uint8_t *out, const fb::FramePlan *plan, uint32_t n,
                                                               const uint64_t *seg_off, const lz4b200_xxh32_state *states,
                                                               uint64_t *frame_off)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    const fb::FramePlan &p = plan[f];
    uint64_t start, o;
    fb::frame_place(p, seg_off, &start, &o);
    for (uint32_t i = 0; i < p.hdr_len; i++) out[start + i] = p.hdr[i];
    for (int b = 0; b < 4; b++) out[o + b] = 0;
    o += 4;
    if (states) {
        const uint32_t h = fw::xxh32_digest(states[f]);
        for (int b = 0; b < 4; b++) out[o + b] = (uint8_t)(h >> (8 * b));
        o += 4;
    }
    frame_off[f] = start;
    if (f == n - 1) frame_off[n] = o;
}

// ---- the frame decoders' group pipeline ---------------------------------------------------------------------------------
// Every frame decoder decodes a frame group by group through the same kernels: arguments, decode, resolve, gather,
// content hash, digest (decode_group).  A group holds the blocks of one or more frames, described by one GroupFrame
// each: the batch decoder's record walk fills one per frame, the group loop (decode_frame_blocks) one per group of a
// frame.  Blocks are indexed frame after frame, the blocks of independent frames first and those of linked frames
// after them.
struct GroupFrame {
    uint64_t in_off;                  // the frame's first byte is at src + in_off (unsigned: payload offsets add to it)
    uint64_t out_off, out_cap;        // the group's output goes to out + out_off, at most out_cap bytes
    uint64_t delivered;               // the frame's bytes that earlier groups delivered
    const fw::FrameWalk *walk;        // the frame's walk
    lz4b200_xxh32_state *content;     // the frame's content hash, carried from group to group (null: hashed by the host)
    lz4b200_frame_result *result;
    uint32_t base, nblocks;           // the group's descriptors of this frame: [base, base + nblocks)
    uint32_t bad;                     // the first of them not delivered: the first to fail its checksum (kNoBlock: none),
                                      // lowered by the resolve step to the first that fails to decode
    uint8_t window;                   // 1: descriptor `base` is a linked window's stored pseudo-block, not output
    uint8_t last;                     // the group ends the frame: the walk status and the EndMark rules apply
};

// ---- batch frame decoder (lz4b200_frame_decompress_batch_device) --------------------------------------------------------
// Many independent frames per call.  Frame f is the one that starts at in + frame_off[f] in a region of frame_len[f]
// bytes.  The host plans groups of whole frames from a count walk; each group's frames are each one group of the
// pipeline above.

// Count walk, one thread per frame: the walk state, the count, and the block count per class (independent blocks at
// nb2[f], linked at nb2[n + f]) for the descriptor scans.
__global__ void __launch_bounds__(128) frame_count_kernel(const uint8_t *in, const uint64_t *frame_off,
                                                          const uint64_t *frame_len, uint32_t n, uint64_t budget,
                                                          fw::FrameWalk *walks, fw::FrameCount *counts, uint32_t *nb2)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    fw::FrameWalk w;
    fw::FrameCount c;
    fw::frame_count(in + frame_off[f], frame_len[f], w, c, budget);
    walks[f] = w;
    counts[f] = c;
    const uint32_t nb = (uint32_t)c.nblocks;                      // the host sends larger frames down the one-frame path
    nb2[f] = c.linked ? 0u : nb;
    nb2[n + f] = c.linked ? nb : 0u;
}

// lz4b200_frame_decoded_bound of the first frame of each region, one thread per region.
__global__ void __launch_bounds__(128) frame_bound_kernel(const uint8_t *in, const uint64_t *frame_off,
                                                          const uint64_t *frame_len, uint32_t n, uint64_t *bound)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    fw::FrameWalk w;
    fw::FrameBlockDesc buf[4];
    uint64_t total = 0;
    while (w.stage != fw::kWalkDone) {
        const uint32_t k = fw::frame_walk(in + frame_off[f], frame_len[f], w, buf, 4);
        for (uint32_t i = 0; i < k; i++)
            total += fw::block_stored(buf[i]) ? fw::block_len(buf[i]) : fw::block_decoded_cap(fw::block_len(buf[i]), w.bs);
    }
    bound[f] = total;
}

// Record walk of the group's frames [f0, f0 + gn), one thread per frame: each frame's descriptors at its base (from the
// scans of the two block-count classes), its block's frame, and its GroupFrame as one group ending the frame.
__global__ void __launch_bounds__(128) frame_record_kernel(const uint8_t *in, const uint64_t *frame_off,
                                                           const uint64_t *frame_len, const uint64_t *frame_out_off,
                                                           const uint64_t *frame_out_cap, uint32_t f0, uint32_t gn,
                                                           const fw::FrameWalk *walks, const fw::FrameCount *counts,
                                                           const uint64_t *scan_ind, const uint64_t *scan_lnk,
                                                           fw::FrameBlockDesc *desc, uint32_t *bframe,
                                                           lz4b200_xxh32_state *states, lz4b200_frame_result *results,
                                                           GroupFrame *frames)
{
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= gn) return;
    const uint32_t f = f0 + g;
    const fw::FrameCount c = counts[f];
    const uint32_t base = (uint32_t)(c.linked ? scan_ind[gn] + scan_lnk[g] : scan_ind[g]);
    fw::FrameWalk w;
    const uint32_t nb = fw::frame_walk(in + frame_off[f], frame_len[f], w, desc + base, (uint32_t)c.nblocks);
    for (uint32_t k = 0; k < nb; k++) bframe[base + k] = g;
    GroupFrame p{};
    p.in_off = frame_off[f];
    p.out_off = frame_out_off[f];
    p.out_cap = frame_out_cap[f];
    p.walk = walks + f;
    p.content = states + g;
    p.result = results + f;
    p.base = base;
    p.nblocks = nb;
    p.bad = fw::kNoBlock;
    p.last = 1;
    frames[g] = p;
}

// Block checksums, one thread per block of the group; frames[g].bad receives the first failing block of frame g.
__global__ void __launch_bounds__(128) frame_batch_checksum_kernel(const uint8_t *in, const fw::FrameBlockDesc *desc,
                                                                   const uint32_t *bframe, uint32_t nb, GroupFrame *frames)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    GroupFrame &p = frames[bframe[b]];
    if (!(p.walk->flg & 0x10)) return;
    if (!fw::block_checksum_ok(in + p.in_off, desc[b])) atomicMin(&p.bad, b - p.base);
}

// The decoder's arguments, one thread per block of the group: blocks at and past a frame's first bad block are not
// decoded (in_len 0, cap 0, like a stored block) and nothing of theirs is delivered.  Linked blocks (index >= nind)
// also get their chain start relative to the linked launch's first block.  slot[b]: the bytes of block b's slot.
__global__ void __launch_bounds__(128) frame_batch_args_kernel(const GroupFrame *frames, const fw::FrameBlockDesc *desc,
                                                               const uint32_t *bframe, uint32_t nb, uint32_t nind,
                                                               uint64_t *in_off, uint32_t *in_len, uint32_t *out_cap,
                                                               uint8_t *pick, uint32_t *link_first, uint32_t *stored_len,
                                                               uint32_t *done, uint32_t *slot)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const GroupFrame &p = frames[bframe[b]];
    const fw::FrameBlockDesc d = desc[b];
    const uint64_t bs = p.walk->bs;
    const bool live = b - p.base < p.bad, stored = fw::block_stored(d), decode = live && !stored;
    in_off[b] = p.in_off + d.payload_off;
    in_len[b] = decode ? fw::block_len(d) : 0u;
    out_cap[b] = decode ? (uint32_t)fw::block_decoded_cap(fw::block_len(d), bs) : 0u;
    pick[b] = decode ? 0 : 1;
    slot[b] = (uint32_t)fw::slot_bytes(fw::block_slot_cap(d, bs));
    if (b >= nind) {
        link_first[b] = p.base - nind;
        stored_len[b] = live && stored ? fw::block_len(d) : 0u;
        done[b] = 0;
    }
}

// One warp per frame of the group: the frame's result after this group, and the gather of its delivered blocks.
// The rules, in order: the first failing block in stream order ends the output; output past out_cap is OUTPUT_FULL
// (nothing of the group delivered), checked before the decode error; then, in the group that ends the frame, the
// walk's status and at the EndMark the content length (the digest kernel compares the content checksum).  hash[g] is
// set when the group's output goes into the frame's content hash (if it has one), which is reset when the frame has
// delivered nothing.  A warp, not a thread: the group loop's one frame may hold thousands of blocks.
__global__ void __launch_bounds__(128) frame_resolve_kernel(GroupFrame *frames, uint32_t gn,
                                                            const fw::FrameBlockDesc *desc, const uint32_t *out_len,
                                                            const int32_t *status, const uint64_t *expected,
                                                            const uint32_t *blk_cap, uint64_t *dst_off, uint32_t *glen,
                                                            uint8_t *hash)
{
    const uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31;
    if (g >= gn) return;                                    // whole warps
    const GroupFrame p = frames[g];
    const uint32_t base = p.base, nrec = p.nblocks, end = min(nrec, p.bad);
    uint32_t good = end;                                    // the first block of [window, end) that failed to decode
    uint64_t total = 0;                                     // the delivered blocks' output, packed in stream order
#pragma unroll 4
    for (uint32_t k0 = 0; k0 < nrec; k0 += 32) {
        const uint32_t k = k0 + lane, b = base + k;
        const bool live = k >= p.window && k < end, stored = live && fw::block_stored(desc[b]);
        const uint32_t m = __ballot_sync(kFull, live && !stored && status[b] != 0);
        if (m && good == end) good = k0 + __ffs(m) - 1;
        const uint32_t len = live && k < good ? (stored ? fw::block_len(desc[b]) : out_len[b]) : 0u;
        uint64_t x = len;
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t y = __shfl_up_sync(kFull, x, d);
            if (lane >= d) x += y;
        }
        if (k < nrec) { dst_off[b] = p.out_off + total + x - len; glen[b] = len; }
        total += __shfl_sync(kFull, x, 31);
    }
    const bool full = total > p.out_cap;
    if (full)
        for (uint32_t k = lane; k < nrec; k += 32) glen[base + k] = 0;
    if (lane) return;
    fw::FrameWalk w = *p.walk;
    if (p.bad != fw::kNoBlock) fw::frame_walk_fail_block(w, desc[base + p.bad], p.bad);
    lz4b200_frame_result r{};
    r.consumed = w.ip;
    r.written = p.delivered;
    if (full) {
        r.status = LZ4B200_FRAME_OUTPUT_FULL;
    } else {
        r.written += total;
        if (good < end) {
            const uint32_t b = base + good;
            r.status = LZ4B200_FRAME_DECOMPRESSION_ERROR;
            r.block_status = status[b];
            if (status[b] == LZ4B200_DEC_OUTPUT_TOO_SMALL) { r.err_expected = expected[b]; r.err_actual = blk_cap[b]; }
            frames[g].bad = good - p.window;
        } else if (p.last && w.status != LZ4B200_OK) {
            r.status = w.status;
        } else if (p.last && w.closed && w.has_size && r.written != w.content_size) {
            r.status = LZ4B200_FRAME_CONTENT_LENGTH;
            r.err_expected = w.content_size;
            r.err_actual = r.written;
        }
    }
    const bool h = p.content && (w.flg & 0x04) && !full;
    if (h && p.delivered == 0) fw::xxh32_reset(*p.content, 0);
    hash[g] = h;
    *p.result = r;
}

// The content hash of the group's output, one CTA per frame, carried in the frame's state; frame_batch_digest_kernel
// then compares the digest at the EndMark.  (The minimum of one CTA per SM lifts the 40-register limit ptxas otherwise
// picks here, which spills.)
__global__ void __launch_bounds__(256, 1) frame_batch_hash_kernel(const uint8_t *out, const GroupFrame *frames,
                                                                  const uint8_t *hash)
{
    __shared__ __align__(16) uint8_t stage[2][kHashChunk + 16];
    const uint32_t g = blockIdx.x;
    if (!hash[g]) return;
    const GroupFrame &p = frames[g];
    content_hash_cta(p.content, out + p.out_off, p.result->written - p.delivered, stage);
}

__global__ void __launch_bounds__(128) frame_batch_digest_kernel(const GroupFrame *frames, uint32_t gn,
                                                                 const uint8_t *hash)
{
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= gn || !hash[g]) return;
    const GroupFrame &p = frames[g];
    const fw::FrameWalk &w = *p.walk;
    if (p.last && p.result->status == LZ4B200_OK && w.closed && w.has_checksum &&
        fw::xxh32_digest(*p.content) != w.content_checksum)
        p.result->status = LZ4B200_FRAME_CONTENT_CHECKSUM;
}

}  // namespace lz4b200

// ---------------------------------------------------------------------------------------------
// host helpers
// ---------------------------------------------------------------------------------------------
namespace {

inline uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline void wr32(uint8_t *p, uint32_t v) { memcpy(p, &v, 4); }

size_t block_size_bytes(int id)
{
    switch (id) {
    case 4: return 64u << 10;
    case 5: return 256u << 10;
    case 6: return 1u << 20;
    case 7: return 4u << 20;
    case 8: return 8u << 20;
    default: return 0;
    }
}

// BlockSize::from_buf_length — frame/header.rs:57-67
int auto_block_size_id(size_t first_write_len)
{
    if (first_write_len > (256u << 10)) return 7;
    if (first_write_len > (64u << 10)) return 5;
    return 4;
}

// Device memory, freed with its owner on the owner's device.  reserve() grows with slack; resize() holds exactly n.
template <typename T> struct DevBuf {
    T *p = nullptr;
    size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { if (p) cudaFree(p); }
    cudaError_t reserve(size_t n) { return n <= cap ? cudaSuccess : resize(n + n / 8 + 256); }
    cudaError_t resize(size_t n)
    {
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&p), n * sizeof(T));
        if (e == cudaSuccess) cap = n; else p = nullptr;
        return e;
    }
};

template <typename T> struct PinnedBuf {
    T *p = nullptr;
    size_t cap = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf &) = delete;
    PinnedBuf &operator=(const PinnedBuf &) = delete;
    ~PinnedBuf() { if (p) cudaFreeHost(p); }
    cudaError_t reserve(size_t n)
    {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        cudaError_t e = cudaHostAlloc(reinterpret_cast<void **>(&p), (n + n / 4 + 64) * sizeof(T), cudaHostAllocDefault);
        if (e == cudaSuccess) cap = n + n / 4 + 64; else p = nullptr;
        return e;
    }
};

constexpr int kMaxLanes = 8;

struct Lane {
    cudaStream_t stream = nullptr;
    cudaEvent_t sizes_ready = nullptr;
    DevBuf<uint8_t> in, slots, out;
    ~Lane()
    {
        if (stream) cudaStreamDestroy(stream);
        if (sizes_ready) cudaEventDestroy(sizes_ready);
    }
};

struct Pipeline {
    Lane lane[kMaxLanes];
    cudaEvent_t desc_ready = nullptr;
    DevBuf<uint32_t> d_tickets;               // kMaxLanes x 8 counters
    PinnedBuf<uint64_t> h_seg;
    PinnedBuf<int32_t> h_status;
    bool ready = false;
    ~Pipeline() { if (desc_ready) cudaEventDestroy(desc_ready); }
};

}  // namespace

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
struct lz4b200_ctx {
    std::unique_ptr<Pipeline> pipe;           // host-batch pipeline state (streams, pinned staging), created on demand
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    DevBuf<uint32_t> d_tickets;               // 3 x {next, retired}
    int dec_ctas_per_sm = 0;
    int enc16s_ctas_per_sm = 0, enc32s_ctas_per_sm = 0;   // split (matcher+emitter) encoder
    int enc_gtab_ctas_per_sm = 0;             // global-table encoder (must reach ENC_GTAB_CTAS)
    int high_priority = 0;                    // lz4b200_ctx_set_priority(ctx, 1): pipeline streams get the highest priority
    DevBuf<uint16_t> d_gtab16;                // global u16 tables (lz4_compress_blocks_gtab / _gtab16)
    const uint32_t *pipe_tickets = nullptr;  // base of the host pipeline's ticket blocks (selects a table region)
    int enc_g16 = 0;                          // LZ4B200_ENC_G16=62|71 (16-lane groups) or 862|871 (8-lane groups): lane-group matchers, 0: off
    int enc_g16_ctas = 8;                     // LZ4B200_ENC_G16_CTAS
    int enc_nib = 0;                          // (A/B build) LZ4B200_ENC_NIB=1..5: shared-memory tags + first-2 verification (gnib / gtagg)
    int enc_nib_ctas = 8;                     // LZ4B200_ENC_NIB_CTAS
    // K1-S2 (one chain per CTA over the TMA-fed ring, lz4b200_solo_kernel.cuh): LZ4B200_ENC_SOLO=2 routes batches of
    // blocks > 64 KiB (and batches of at most enc_solo_small_max small blocks) to it
    int enc_solo = 0, enc_solo_ctas_per_sm = 0, enc_solo2_ctas_per_sm = 0;
    uint32_t enc_solo_small_max = 0;
#ifdef LZ4B200_AB_VARIANTS
    int enc16_ctas_per_sm = 0, enc32_ctas_per_sm = 0;
    int enc_gtab = 71;                        // LZ4B200_ENC_GTAB=10*matchers+emitters per CTA (62|71|44|151)
    DevBuf<uint16_t> d_ttab16;                // K1-T tables
    DevBuf<uint32_t> d_gtag32;                // tagged global tables (lz4_compress_blocks_gtag)
    int enc_gtag = 0;                         // LZ4B200_ENC_GTAG=71|62: tagged entries (measured slower)
    int enc_gtag_ctas = 8;
    int enc_single_warp = 0;                  // LZ4B200_ENC_SINGLE_WARP=1: one warp searches and emits
    int dec_ctas_override = 0;                // LZ4B200_DEC_CTAS=n CTAs per SM
    int dec_conv = 0;                         // LZ4B200_DEC_CONV=1: warp-converged decoder loop
    int dec_batched = 0;                      // LZ4B200_DEC_BATCHED=1
    int dec_group_override = 0;               // LZ4B200_DEC_GROUP=4|8|16|32
    // K1-T / K2-T (one block per thread, lz4b200_thread_kernels.cuh)
    uint32_t enc_thread_min = 0xffffffffu, dec_thread_min = 0xffffffffu;
    int enc_thread_lanes = 0, dec_thread_lanes = 0;
    uint32_t enc_thread_max = 16384, dec_thread_max = 65536;
#endif
    std::string last_error;
    const char *last_kernel[2] = {"", ""};   // what the launchers picked last: [0] compress, [1] decompress (for the bench record)
    std::string last_kernel_both;             // storage of last_kernel[0] when the u16 and u32 encoders both ran
    uint32_t range_nb = 0;                    // lz4b200_frame_range_compress -> _pack hand-over
    const uint8_t *range_in = nullptr;
    size_t frame_budget = 256u << 20;         // device bytes the frame decoder's block slots / staged input may take per group

    // scratch for host-pointer and frame entry points
    DevBuf<uint8_t> d_in, d_out, d_slots, d_flags, d_pick, d_dict;
    DevBuf<uint64_t> d_in_off, d_out_off, d_seg_off, d_expected, d_off_b;
    DevBuf<uint32_t> d_in_len, d_out_cap, d_out_len, d_info, d_seg_size, d_payload_len, d_link_first, d_stored_len, d_done;
    DevBuf<int32_t> d_status;
    // device-resident frame decoder: walk state, the block descriptors of one walk launch, the first block whose
    // checksum fails, the running content hash, and the group loop's result
    DevBuf<fw::FrameWalk> d_walk;
    DevBuf<fw::FrameBlockDesc> d_desc;
    DevBuf<uint32_t> d_bad;
    DevBuf<lz4b200_xxh32_state> d_content;
    DevBuf<lz4b200_frame_result> d_result;
    // batch frame decoder: per frame the walk, the count and the two block counts; per group the scans and the hash
    // flags; per block its frame, slot bytes and gather lengths
    DevBuf<fw::FrameWalk> d_fwalk;
    DevBuf<fw::FrameCount> d_fcount;
    DevBuf<uint32_t> d_fnb, d_bframe, d_bslot, d_glen;
    DevBuf<uint64_t> d_fscan, d_gdst;
    DevBuf<uint8_t> d_fhash;
    DevBuf<GroupFrame> d_gframe;              // the frames of a decode group
    DevBuf<fb::FramePlan> d_fplan;            // batch frame encoder: the host's plan, one entry per frame
    // frame index and range decode: per block a linked block's reach; per range of a chunk its first block, block count
    // and item offset; per item of a window the length its block must decode to.  Linked frames: the touched blocks'
    // difference array, a window's marker entries, blocks and pieces, the carry from window to window, and per segment
    // of a round whether a requested byte stayed unresolved
    DevBuf<uint32_t> d_reach, d_rfirst, d_rcount, d_rwant;
    DevBuf<uint64_t> d_ritem;
    DevBuf<int32_t> d_rtouch;
    DevBuf<uint32_t> d_rent, d_rcarry, d_rflag;
    DevBuf<fr::MarkBlock> d_rblk;
    DevBuf<fr::MarkPiece> d_rpiece;
    uint64_t last_range_blocks = 0;           // block decodes of the last ranges call (lz4b200_ctx_last_range_blocks)

    bool check(cudaError_t e, const char *what)
    {
        if (e == cudaSuccess) return true;
        last_error = std::string(what) + ": " + cudaGetErrorString(e);
        return false;
    }

    __attribute__((visibility("hidden"))) ~lz4b200_ctx()     // not part of the library's exports
    {
        if (stream) cudaStreamSynchronize(stream);
        if (pipe)
            for (const Lane &l : pipe->lane)
                if (l.stream) cudaStreamSynchronize(l.stream);
        if (stream) cudaStreamDestroy(stream);
    }
};

namespace {

#ifdef LZ4B200_AB_VARIANTS
constexpr int kEnc16Warps = 4;     // v1 encoder: 8 KiB table per warp
constexpr int kEnc32Warps = 2;     // 2 x 16 KiB tables per CTA
#endif
#ifndef ENC16_PAIRS
#define ENC16_PAIRS 3
#endif
// Shape of the global-table encoder lz4_compress_blocks_gtab<u16, M, E, SMEM, CTAS>: M matcher warps and E emitter warps
// per CTA, CTAS CTAs per SM (which also sets the register budget).  The first SMEM matchers of a CTA keep their 8 KiB
// table in shared memory, the other M - SMEM in global memory, where every SM's tables share the 50 MB L2 of an H100
// with the streaming input and output.  The default keeps all 21 tables of an SM in shared memory (183 KB with the
// queues): no table traffic reaches L2, and the 60 KB of L1 left beside them still caches the input.  On one H100 at
// 400 W it compresses 1 GiB of 64 KiB JSON blocks in 25 % less time than the same shape with global tables; more chains
// per SM with part of the tables in global memory, or a larger shared-memory carveout that shrinks L1 to 28 KB, are
// slower (DESIGN.md §6).
#ifndef ENC_GTAB_M
#define ENC_GTAB_M 7
#endif
#ifndef ENC_GTAB_E
#define ENC_GTAB_E 1
#endif
#ifndef ENC_GTAB_SMEM
#define ENC_GTAB_SMEM 7
#endif
#ifndef ENC_GTAB_CTAS
#define ENC_GTAB_CTAS 3
#endif
constexpr int kGtabM = ENC_GTAB_M, kGtabE = ENC_GTAB_E, kGtabSmem = ENC_GTAB_SMEM, kGtabCtasPerSm = ENC_GTAB_CTAS;
constexpr int kGtabSmemBytes = kGtabSmem * 4096 * (int)sizeof(uint16_t);
static_assert(kGtabSmem >= 0 && kGtabSmem <= kGtabM, "ENC_GTAB_SMEM: at most ENC_GTAB_M shared-memory tables");
#define LZ4B200_STR2(x) #x
#define LZ4B200_STR(x) LZ4B200_STR2(x)
constexpr const char *kGtabKernelName = "lz4_compress_blocks_gtab<unsigned short, " LZ4B200_STR(ENC_GTAB_M) ", " LZ4B200_STR(ENC_GTAB_E)
                                        ", " LZ4B200_STR(ENC_GTAB_SMEM) ", " LZ4B200_STR(ENC_GTAB_CTAS) ">";
constexpr int kEnc16Pairs = ENC16_PAIRS;   // split encoder: matcher+emitter pairs per CTA (named barriers: <= 3)
constexpr int kEnc32Pairs = 2;

#define CTX_CUDA(ctx, call)                                              \
    do {                                                                 \
        if (!(ctx)->check((call), #call)) return LZ4B200_CUDA_ERROR;     \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

template <int G>
lz4b200_status launch_decompress_g(lz4b200_ctx *ctx, const BatchArgs &a, cudaStream_t s)
{
    const uint32_t per_cta = kDecWarpsPerCta * (32 / G);
    uint32_t want = (a.nblocks + per_cta - 1) / per_cta;
    uint32_t grid = std::min<uint32_t>(want, (uint32_t)(ctx->sm_count * std::min(32, 64 / kDecWarpsPerCta)));   // 64 warps per SM
#ifdef LZ4B200_AB_VARIANTS
    if (ctx->dec_ctas_override) grid = std::min<uint32_t>(want, (uint32_t)(ctx->sm_count * ctx->dec_ctas_override));
    if (!a.dict_len && ctx->dec_conv) { lz4_decompress_blocks_conv<G><<<grid, kDecWarpsPerCta * 32, 0, s>>>(a); CTX_CUDA(ctx, cudaGetLastError()); return LZ4B200_OK; }
    if (!a.dict_len && ctx->dec_batched) { lz4_decompress_blocks<G, 1, false><<<grid, kDecWarpsPerCta * 32, 0, s>>>(a); CTX_CUDA(ctx, cudaGetLastError()); return LZ4B200_OK; }
#endif
    const uint32_t warps = (a.nblocks + (32 / G) - 1) / (32 / G);
    const bool one_warp = !a.dict_len && kDecWarpsPerCta > 1 && warps <= (uint32_t)ctx->sm_count * 32u;   // all resident as one-warp CTAs
    if (one_warp) lz4_decompress_blocks<G, 0, false, 1><<<warps, 32, 0, s>>>(a);
    else if (a.dict_len) lz4_decompress_blocks<G, 0, true><<<grid, kDecWarpsPerCta * 32, 0, s>>>(a);
    else lz4_decompress_blocks<G, 0, false><<<grid, kDecWarpsPerCta * 32, 0, s>>>(a);
#define LZ4B200_DEC_NAME(g, d, w) "lz4_decompress_blocks<" #g ", 0, " #d ", " w ">"
    ctx->last_kernel[1] = one_warp ? (G == 8 ? LZ4B200_DEC_NAME(8, 0, "1") : G == 16 ? LZ4B200_DEC_NAME(16, 0, "1") : LZ4B200_DEC_NAME(32, 0, "1"))
        : a.dict_len ? (G == 8 ? LZ4B200_DEC_NAME(8, 1, LZ4B200_STR(DEC_WARPS_PER_CTA)) : G == 16 ? LZ4B200_DEC_NAME(16, 1, LZ4B200_STR(DEC_WARPS_PER_CTA)) : LZ4B200_DEC_NAME(32, 1, LZ4B200_STR(DEC_WARPS_PER_CTA)))
                     : (G == 8 ? LZ4B200_DEC_NAME(8, 0, LZ4B200_STR(DEC_WARPS_PER_CTA)) : G == 16 ? LZ4B200_DEC_NAME(16, 0, LZ4B200_STR(DEC_WARPS_PER_CTA)) : LZ4B200_DEC_NAME(32, 0, LZ4B200_STR(DEC_WARPS_PER_CTA)));
#undef LZ4B200_DEC_NAME
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}

// Lanes per block: with few blocks every block gets a whole warp (widest copies, most parallel
// chains); with many blocks narrower groups cut the warp-instructions per sequence.
int pick_dec_group(const lz4b200_ctx *ctx, uint32_t nblocks)
{
#ifdef LZ4B200_AB_VARIANTS
    if (ctx->dec_group_override) return ctx->dec_group_override;
#endif
    (void)ctx;
    // narrower groups win on large batches of 64 KiB JSON blocks (fewer warp-instructions per sequence); whole warps win
    // when there are too few blocks to fill the GPU
    if (nblocks >= 12288) return 8;
    return nblocks >= 4096 ? 16 : 32;
}

#ifdef LZ4B200_AB_VARIANTS
// Active lanes per warp for the thread-per-block kernels: a batch with fewer blocks than the GPU has lanes is
// spread over more warps.
int pick_thread_lanes(const lz4b200_ctx *ctx, uint32_t threads, int override_lanes)
{
    if (override_lanes == 8 || override_lanes == 16 || override_lanes == 32) return override_lanes;
    const uint32_t full = (uint32_t)ctx->sm_count * 64u * 32u;      // every lane of every resident warp
    if (threads * 4u <= full) return 8;
    return threads * 2u <= full ? 16 : 32;
}

template <int kLanes>
lz4b200_status launch_decompress_thread(lz4b200_ctx *ctx, const BatchArgs &a, uint32_t threads, cudaStream_t s)
{
    const uint32_t per_cta = kThreadCtaWarps * kLanes;
    lz4_decompress_blocks_thread<kLanes><<<(threads + per_cta - 1) / per_cta, kThreadCtaWarps * 32, 0, s>>>(a);
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}
#endif

lz4b200_status launch_decompress(lz4b200_ctx *ctx, const BatchArgs &args, cudaStream_t s, uint32_t *tickets = nullptr)
{
    if (args.nblocks == 0) return LZ4B200_OK;
    BatchArgs a = args;
    a.tickets = tickets ? tickets : ctx->d_tickets.p;
#ifdef LZ4B200_AB_VARIANTS
    if (!a.dict_len && a.nblocks >= ctx->dec_thread_min) {
        const uint32_t threads = std::min(a.nblocks, ctx->dec_thread_max);
        switch (pick_thread_lanes(ctx, threads, ctx->dec_thread_lanes)) {
        case 8: return launch_decompress_thread<8>(ctx, a, threads, s);
        case 16: return launch_decompress_thread<16>(ctx, a, threads, s);
        default: return launch_decompress_thread<32>(ctx, a, threads, s);
        }
    }
    if (pick_dec_group(ctx, a.nblocks) == 4) return launch_decompress_g<4>(ctx, a, s);
#endif
    switch (pick_dec_group(ctx, a.nblocks)) {
    case 8: return launch_decompress_g<8>(ctx, a, s);
    case 16: return launch_decompress_g<16>(ctx, a, s);
    default: return launch_decompress_g<32>(ctx, a, s);
    }
}

// One table region per concurrently running launch (the host pipeline launches from up to 8 lanes): the ticket block
// doubles as the region selector.
static size_t table_slot(const lz4b200_ctx *ctx, const uint32_t *tickets)
{
    return tickets == ctx->d_tickets.p ? 0 : 1 + ((size_t)(tickets - ctx->pipe_tickets) / 8u) % 8u;
}

#ifdef LZ4B200_AB_VARIANTS
// The measured-and-rejected K1 variants (DESIGN.md §6).  Returns true when one of them took the batch.
static bool launch_compress_variant(lz4b200_ctx *ctx, const BatchArgs &a, uint32_t max_in_len, cudaStream_t s, uint32_t *tickets,
                                    lz4b200_status *st)
{
    *st = LZ4B200_OK;
    if (a.dict_len) return false;
    if (ctx->enc_solo == 1 && max_in_len != 0 && (max_in_len > 65536u || a.nblocks <= ctx->enc_solo_small_max)) {
        const uint32_t grid = std::min<uint32_t>(a.nblocks, (uint32_t)(ctx->sm_count * ctx->enc_solo_ctas_per_sm));
        lz4_compress_blocks_solo<<<grid, 64, kSoloSmemBytes, s>>>(a, tickets + 4);
        if (!ctx->check(cudaGetLastError(), "solo launch")) *st = LZ4B200_CUDA_ERROR;
        return true;
    }
    if (max_in_len != 0 && max_in_len <= 65536u && a.nblocks >= ctx->enc_thread_min) {
        // K1-T: one block per thread, 8 KiB table per thread in global memory
        const uint32_t threads = std::min(a.nblocks, ctx->enc_thread_max);
        const size_t region = (size_t)ctx->enc_thread_max * 4096u;                  // u16 entries
        const size_t slot = table_slot(ctx, tickets);
        if (!ctx->check(ctx->d_ttab16.reserve(region * (slot ? 9u : 1u)), "thread tables")) { *st = LZ4B200_CUDA_ERROR; return true; }
        uint16_t *gt = ctx->d_ttab16.p + slot * region;
        const int lanes = pick_thread_lanes(ctx, threads, ctx->enc_thread_lanes);
        const uint32_t per_cta = kThreadCtaWarps * lanes, grid = (threads + per_cta - 1) / per_cta;
        if (lanes == 8) lz4_compress_blocks_thread<8><<<grid, kThreadCtaWarps * 32, 0, s>>>(a, tickets + 2, gt);
        else if (lanes == 16) lz4_compress_blocks_thread<16><<<grid, kThreadCtaWarps * 32, 0, s>>>(a, tickets + 2, gt);
        else lz4_compress_blocks_thread<32><<<grid, kThreadCtaWarps * 32, 0, s>>>(a, tickets + 2, gt);
        if (!ctx->check(cudaGetLastError(), "thread launch")) *st = LZ4B200_CUDA_ERROR;
        return true;
    }
    if (max_in_len != 0 && max_in_len <= 65536u && a.nblocks > (uint32_t)ctx->sm_count * 24u) {
        const size_t slot = table_slot(ctx, tickets);
        if (ctx->enc_gtag) {                                                         // tagged (tag, position) entries
            const int m = ctx->enc_gtag / 10;
            const uint32_t grid = std::min<uint32_t>((a.nblocks + m - 1) / m, (uint32_t)(ctx->sm_count * ctx->enc_gtag_ctas));
            const size_t region = (size_t)ctx->sm_count * 8u * 8u * 4096u;
            if (!ctx->check(ctx->d_gtag32.reserve(region * 9u), "gtag")) { *st = LZ4B200_CUDA_ERROR; return true; }
            uint32_t *gt = ctx->d_gtag32.p + slot * region;
            if (m == 6) lz4_compress_blocks_gtag<6, 2><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
            else lz4_compress_blocks_gtag<7, 1><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
            if (!ctx->check(cudaGetLastError(), "gtag launch")) *st = LZ4B200_CUDA_ERROR;
            return true;
        }
        const int m = ctx->enc_gtab / 10, e = ctx->enc_gtab % 10;
        if (ctx->enc_gtab && (m != 7 || e != 1)) {                                   // other global-table CTA shapes
            const uint32_t grid = std::min<uint32_t>((a.nblocks + m - 1) / m, (uint32_t)ctx->sm_count * (m == 15 ? 4u : 8u));
            const size_t region = (size_t)ctx->sm_count * 8u * 28u * 4096u;
            if (!ctx->check(ctx->d_gtab16.reserve(region * 9u), "gtab")) { *st = LZ4B200_CUDA_ERROR; return true; }
            uint16_t *gt = ctx->d_gtab16.p + slot * region;
            if (m == 15) lz4_compress_blocks_gtab<uint16_t, 15, 1, 0><<<grid, 512, 0, s>>>(a, tickets + 2, gt);
            else if (m == 6 && e == 2) lz4_compress_blocks_gtab<uint16_t, 6, 2, 0><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
            else if (m == 4 && e == 4) lz4_compress_blocks_gtab<uint16_t, 4, 4, 0><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
            else return false;
            if (!ctx->check(cudaGetLastError(), "gtab launch")) *st = LZ4B200_CUDA_ERROR;
            return true;
        }
    }
    if (ctx->enc_single_warp) {                                                      // v1: one warp searches and emits
        if (max_in_len == 0 || max_in_len <= 65536u) {
            const uint32_t grid = std::min<uint32_t>((a.nblocks + kEnc16Warps - 1) / kEnc16Warps, (uint32_t)ctx->sm_count * (uint32_t)ctx->enc16_ctas_per_sm);
            lz4_compress_blocks<uint16_t, kEnc16Warps><<<grid, kEnc16Warps * 32, kEnc16Warps * 4096 * sizeof(uint16_t), s>>>(a, tickets + 2);
        }
        if (max_in_len == 0 || max_in_len > 65536u) {
            const uint32_t grid = std::min<uint32_t>((a.nblocks + kEnc32Warps - 1) / kEnc32Warps, (uint32_t)(ctx->sm_count * ctx->enc32_ctas_per_sm));
            lz4_compress_blocks<uint32_t, kEnc32Warps><<<grid, kEnc32Warps * 32, kEnc32Warps * 4096 * sizeof(uint32_t), s>>>(a, tickets + 4);
        }
        if (!ctx->check(cudaGetLastError(), "v1 launch")) *st = LZ4B200_CUDA_ERROR;
        return true;
    }
    return false;
}
#endif

// K1 launcher.  Blocks <= 64 KiB: u16 tables; larger: u32 tables; unknown mix (max_in_len == 0): both kernels run over
// the same ticket space and each skips the other's blocks.
//   many small blocks (> 24 per SM, no dictionary)  -> gtab: 7 matchers per emitter, ENC_GTAB_* shape (21 chains per SM,
//                                                      tables in shared memory; lane-group matchers: more, global tables)
//   fewer / dictionary                              -> shared-memory tables, matcher + emitter pairs
//   blocks > 64 KiB without dictionary              -> one chain per CTA over the TMA-fed ring when enabled
lz4b200_status launch_compress(lz4b200_ctx *ctx, const BatchArgs &args, uint32_t max_in_len, cudaStream_t s,
                               uint32_t *tickets = nullptr)
{
    if (!tickets) tickets = ctx->d_tickets.p;
    if (args.nblocks == 0) return LZ4B200_OK;
    const BatchArgs &a = args;
#ifdef LZ4B200_AB_VARIANTS
    {
        lz4b200_status vst;
        if (launch_compress_variant(ctx, a, max_in_len, s, tickets, &vst)) return vst;
    }
#endif
    if (!a.dict_len && ctx->enc_solo == 2 && max_in_len != 0 && (max_in_len > 65536u || a.nblocks <= ctx->enc_solo_small_max)) {
        const uint32_t grid = std::min<uint32_t>(a.nblocks, (uint32_t)(ctx->sm_count * ctx->enc_solo2_ctas_per_sm));
        lz4_compress_blocks_solo2<<<grid, 64, kSolo2SmemBytes, s>>>(a, tickets + 4);
        ctx->last_kernel[0] = "lz4_compress_blocks_solo2";
        CTX_CUDA(ctx, cudaGetLastError());
        return LZ4B200_OK;
    }
    {                                                       // u16 tables: every block with input (+ dictionary) <= 64 KiB
        if (!a.dict_len && a.nblocks > (uint32_t)ctx->sm_count * 24u) {
            // u16 entries: tables of 4096 for the CTAs per SM x chains per CTA that keep them in global memory, one region
            // per concurrently running launch
            const int g16_m = (ctx->enc_g16 % 100) / 10, g16_g = ctx->enc_g16 >= 800 ? 8 : 16;
            const size_t chains_per_sm = ctx->enc_g16 ? (size_t)ctx->enc_g16_ctas * (32 / g16_g) * g16_m : (ctx->enc_nib >= 4 ? 112u : ctx->enc_nib ? 8u * 7u : (size_t)kGtabCtasPerSm * (kGtabM - kGtabSmem));   // enc_nib: A/B build only
            const size_t region = (size_t)ctx->sm_count * chains_per_sm * 4096u;
            if (!ctx->check(ctx->d_gtab16.reserve(region * 9u), "gtab")) return LZ4B200_CUDA_ERROR;
            uint16_t *gt = ctx->d_gtab16.p + table_slot(ctx, tickets) * region;
#ifdef LZ4B200_AB_VARIANTS
            if (ctx->enc_nib && !ctx->enc_g16) {                                     // tags in shared memory: 1 = nibbles x 8 CTAs, 2 = bytes x 6 CTAs, 3 = nibbles x 6 CTAs (40 registers)
                const uint32_t ctas = std::min(ctx->enc_nib_ctas, ctx->enc_nib == 1 ? 8 : 6);
                const uint32_t grid = std::min<uint32_t>((a.nblocks + 6) / 7, (uint32_t)ctx->sm_count * ctas);
                if (ctx->enc_nib == 4) {                                             // lane groups of 8 + 2-bit tags: 4 x 28 chains per SM
                    const uint32_t g4 = std::min<uint32_t>((a.nblocks + 27) / 28, (uint32_t)ctx->sm_count * std::min(ctx->enc_nib_ctas, 4));
                    lz4_compress_blocks_gtagg<8, 7, 1, 2, 4><<<g4, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtagg<8, 7, 1, 2, 4>";
                } else if (ctx->enc_nib == 5) {                                      // lane groups of 16 + 2-bit tags: 8 x 14 chains per SM
                    const uint32_t g5 = std::min<uint32_t>((a.nblocks + 13) / 14, (uint32_t)ctx->sm_count * std::min(ctx->enc_nib_ctas, 8));
                    lz4_compress_blocks_gtagg<16, 7, 1, 2, 8><<<g5, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtagg<16, 7, 1, 2, 8>";
                } else
                if (ctx->enc_nib == 2) { lz4_compress_blocks_gnib<7, 1, 8, 6><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gnib<7, 1, 8, 6>"; }
                else if (ctx->enc_nib == 3) { lz4_compress_blocks_gnib<7, 1, 4, 6><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gnib<7, 1, 4, 6>"; }
                else { lz4_compress_blocks_gnib<7, 1, 4, 8><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gnib<7, 1, 4, 8>"; }
            } else
#endif
            if (ctx->enc_g16) {                                               // 2 or 4 chains per matcher warp
                const int m = (ctx->enc_g16 % 100) / 10, gsz = ctx->enc_g16 >= 800 ? 8 : 16;   // 62 | 71 (G = 16), 862 | 871 (G = 8)
                const int per_cta = (32 / gsz) * m;
                const uint32_t grid = std::min<uint32_t>((a.nblocks + per_cta - 1) / per_cta, (uint32_t)(ctx->sm_count * ctx->enc_g16_ctas));
                if (gsz == 8 && m == 7) { lz4_compress_blocks_gtabg<8, 7, 1><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtabg<8, 7, 1>"; }
                else if (gsz == 8) { lz4_compress_blocks_gtabg<8, 6, 2><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtabg<8, 6, 2>"; }
                else if (m == 7) { lz4_compress_blocks_gtabg<16, 7, 1><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtabg<16, 7, 1>"; }
                else { lz4_compress_blocks_gtabg<16, 6, 2><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtabg<16, 6, 2>"; }
            } else {
                const uint32_t grid = std::min<uint32_t>((a.nblocks + kGtabM - 1) / kGtabM, (uint32_t)ctx->sm_count * kGtabCtasPerSm);
                lz4_compress_blocks_gtab<uint16_t, kGtabM, kGtabE, kGtabSmem, kGtabCtasPerSm>
                    <<<grid, (kGtabM + kGtabE) * 32, kGtabSmemBytes, s>>>(a, tickets + 2, gt);
                ctx->last_kernel[0] = kGtabKernelName;
            }
        } else {
            ctx->last_kernel[0] = a.dict_len ? "lz4_compress_blocks_split<unsigned short, " LZ4B200_STR(ENC16_PAIRS) ", 1>"
                                             : "lz4_compress_blocks_split<unsigned short, " LZ4B200_STR(ENC16_PAIRS) ", 0>";
            const uint32_t grid = std::min<uint32_t>((a.nblocks + kEnc16Pairs - 1) / kEnc16Pairs, (uint32_t)(ctx->sm_count * ctx->enc16s_ctas_per_sm));
            if (a.dict_len)
                lz4_compress_blocks_split<uint16_t, kEnc16Pairs, true>
                    <<<grid, kEnc16Pairs * 64, split_smem_bytes<uint16_t, kEnc16Pairs>(), s>>>(a, tickets + 2);
            else
                lz4_compress_blocks_split<uint16_t, kEnc16Pairs, false>
                    <<<grid, kEnc16Pairs * 64, split_smem_bytes<uint16_t, kEnc16Pairs>(), s>>>(a, tickets + 2);
        }
        CTX_CUDA(ctx, cudaGetLastError());
    }
    if (max_in_len == 0 || (uint64_t)max_in_len + a.dict_len > 65536u) {
        // a bound above 64 KiB names the large-block kernel alone; an unknown bound, or a dictionary that takes the span
        // above 64 KiB, leaves work for both kernels, and the record names both in launch order
        static_assert(kEnc32Pairs == 2, "the kernel names below spell out kEnc32Pairs");
        const char *k32 = a.dict_len ? "lz4_compress_blocks_split<unsigned int, 2, 1>" : "lz4_compress_blocks_split<unsigned int, 2, 0>";
        if (max_in_len > 65536u) {
            ctx->last_kernel[0] = k32;
        } else {
            ctx->last_kernel_both = std::string(ctx->last_kernel[0]) + " + " + k32;
            ctx->last_kernel[0] = ctx->last_kernel_both.c_str();
        }
        const uint32_t grid = std::min<uint32_t>((a.nblocks + kEnc32Pairs - 1) / kEnc32Pairs, (uint32_t)(ctx->sm_count * ctx->enc32s_ctas_per_sm));
        if (a.dict_len)
            lz4_compress_blocks_split<uint32_t, kEnc32Pairs, true>
                <<<grid, kEnc32Pairs * 64, split_smem_bytes<uint32_t, kEnc32Pairs>(), s>>>(a, tickets + 4);
        else
            lz4_compress_blocks_split<uint32_t, kEnc32Pairs, false>
                <<<grid, kEnc32Pairs * 64, split_smem_bytes<uint32_t, kEnc32Pairs>(), s>>>(a, tickets + 4);
        CTX_CUDA(ctx, cudaGetLastError());
    }
    return LZ4B200_OK;
}

// The reference keeps only the last WINDOW_SIZE bytes of a dictionary (init_dict, compress.rs:571-575) and drops
// dictionaries of <= 3 bytes (compress_into_vec_with_dict, compress.rs:626-628).
void normalize_dict(const uint8_t *&dict, size_t &dict_len, bool for_compress)
{
    if (!dict || (for_compress && dict_len <= 3)) { dict = nullptr; dict_len = 0; return; }
    if (dict_len > 65536) { dict += dict_len - 65536; dict_len = 65536; }
}

// The batch's dictionary, normalised, in a.
void set_dict(BatchArgs &a, const uint8_t *dict, size_t dict_len, bool for_compress)
{
    normalize_dict(dict, dict_len, for_compress);
    a.dict = dict;
    a.dict_len = (uint32_t)dict_len;
}

}  // namespace

extern "C" {

int lz4b200_abi_version(void) { return LZ4B200_ABI_VERSION; }

int lz4b200_host_pointer_kind(const void *p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return -1; }
    return (int)a.type;                       // 0 unregistered (pageable), 1 host (pinned), 2 device, 3 managed
}

const char *lz4b200_status_string(int s)
{
    switch (s) {
    case LZ4B200_OK: return "ok";
    case LZ4B200_COMPRESS_OUTPUT_TOO_SMALL:
        return "output is too small for the compressed data, use get_maximum_output_size to reserve enough space";
    case LZ4B200_DEC_OUTPUT_TOO_SMALL: return "provided output is too small for the decompressed data";
    case LZ4B200_DEC_LITERAL_OUT_OF_BOUNDS: return "literal is out of bounds of the input";
    case LZ4B200_DEC_EXPECTED_ANOTHER_BYTE: return "expected another byte, found none";
    case LZ4B200_DEC_OFFSET_ZERO: return "0 is not a valid match offset";
    case LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS: return "the offset to copy is not contained in the decompressed buffer";
    case LZ4B200_FRAME_DECOMPRESSION_ERROR: return "frame: block decompression error";
    case LZ4B200_FRAME_WRONG_MAGIC: return "frame: wrong magic number";
    case LZ4B200_FRAME_RESERVED_BITS: return "frame: reserved bits set";
    case LZ4B200_FRAME_UNSUPPORTED_VERSION: return "frame: unsupported version";
    case LZ4B200_FRAME_UNSUPPORTED_BLOCKSIZE: return "frame: unsupported block size";
    case LZ4B200_FRAME_HEADER_CHECKSUM: return "frame: header checksum error";
    case LZ4B200_FRAME_BLOCK_CHECKSUM: return "frame: block checksum error";
    case LZ4B200_FRAME_CONTENT_CHECKSUM: return "frame: content checksum error";
    case LZ4B200_FRAME_CONTENT_LENGTH: return "frame: content length differs from the header";
    case LZ4B200_FRAME_BLOCK_TOO_BIG: return "frame: block too big";
    case LZ4B200_FRAME_SKIPPABLE: return "frame: skippable frame";
    case LZ4B200_FRAME_DICTIONARY: return "frame: dictionaries are not supported";
    case LZ4B200_FRAME_IO_EOF: return "frame: unexpected end of input";
    case LZ4B200_FRAME_LINKED_UNSUPPORTED: return "frame: linked blocks are not supported on the GPU path";
    case LZ4B200_FRAME_OUTPUT_FULL: return "frame: output buffer exhausted";
    case LZ4B200_INVALID_ARGUMENT: return "invalid argument";
    case LZ4B200_CUDA_ERROR: return "CUDA error";
    default: return "unknown status";
    }
}

const char *lz4b200_last_cuda_error(const lz4b200_ctx *ctx) { return ctx ? ctx->last_error.c_str() : ""; }

lz4b200_status lz4b200_ctx_create(int device, lz4b200_ctx **out)
{
    if (!out) return LZ4B200_INVALID_ARGUMENT;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return LZ4B200_CUDA_ERROR;
    lz4b200_ctx *ctx = new lz4b200_ctx();
    ctx->device = device;
    DeviceGuard guard(device);
    bool ok = ctx->check(cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device), "sm count") &&
              ctx->check(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking), "stream") &&
              ctx->check(ctx->d_tickets.resize(8), "tickets") &&
              ctx->check(cudaMemset(ctx->d_tickets.p, 0, 8 * sizeof(uint32_t)), "tickets memset");
    if (ok) {
        ok = ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->dec_ctas_per_sm, lz4_decompress_blocks<8, 0, false>,
                                                                      kDecWarpsPerCta * 32, 0), "occupancy dec") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                            &ctx->enc16s_ctas_per_sm, lz4_compress_blocks_split<uint16_t, kEnc16Pairs, false>, kEnc16Pairs * 64,
                            split_smem_bytes<uint16_t, kEnc16Pairs>()), "occupancy enc16 split") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                            &ctx->enc32s_ctas_per_sm, lz4_compress_blocks_split<uint32_t, kEnc32Pairs, false>, kEnc32Pairs * 64,
                            split_smem_bytes<uint32_t, kEnc32Pairs>()), "occupancy enc32 split") &&
             ctx->check(cudaFuncSetAttribute(lz4_compress_blocks_solo2, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)kSolo2SmemBytes), "solo2 smem") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->enc_solo2_ctas_per_sm, lz4_compress_blocks_solo2, 64,
                                                                      kSolo2SmemBytes), "occupancy solo2");
        // The global-table encoder's register budget and table region assume ENC_GTAB_CTAS resident CTAs per SM.  Its
        // carveout is the least shared memory those CTAs need (the driver rounds up to the next supported size): the rest
        // of the SM's 256 KB stays L1, which caches the input bytes every probe and extension reads.
        auto *gtab = lz4_compress_blocks_gtab<uint16_t, kGtabM, kGtabE, kGtabSmem, kGtabCtasPerSm>;
        cudaFuncAttributes fa{};
        int smem_sm = 0, smem_reserved = 0;
        ok = ok && ctx->check(cudaFuncGetAttributes(&fa, gtab), "gtab attributes") &&
             ctx->check(cudaDeviceGetAttribute(&smem_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, device), "smem per SM") &&
             ctx->check(cudaDeviceGetAttribute(&smem_reserved, cudaDevAttrReservedSharedMemoryPerBlock, device), "reserved smem");
        if (ok) {
            const size_t need = (size_t)kGtabCtasPerSm * (fa.sharedSizeBytes + kGtabSmemBytes + smem_reserved);
            const int carveout = (int)std::min<size_t>(100, (need * 100 + smem_sm - 1) / std::max(1, smem_sm));
            ok = ctx->check(cudaFuncSetAttribute(gtab, cudaFuncAttributeMaxDynamicSharedMemorySize, kGtabSmemBytes), "gtab smem") &&
                 ctx->check(cudaFuncSetAttribute(gtab, cudaFuncAttributePreferredSharedMemoryCarveout, carveout), "gtab carveout") &&
                 ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->enc_gtab_ctas_per_sm, gtab, (kGtabM + kGtabE) * 32,
                                                                          kGtabSmemBytes), "occupancy gtab");
            if (getenv("LZ4B200_DEBUG"))
                fprintf(stderr, "lz4b200: %s: %zu bytes of shared memory per SM, carveout %d %%\n", kGtabKernelName, need, carveout);
        }
        ctx->enc_solo_small_max = (uint32_t)(ctx->sm_count * std::max(1, ctx->enc_solo2_ctas_per_sm));
    }
#ifdef LZ4B200_AB_VARIANTS
    if (ok) {
        ok = ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                            &ctx->enc16_ctas_per_sm, lz4_compress_blocks<uint16_t, kEnc16Warps>, kEnc16Warps * 32,
                            kEnc16Warps * 4096 * sizeof(uint16_t)), "occupancy enc16") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                            &ctx->enc32_ctas_per_sm, lz4_compress_blocks<uint32_t, kEnc32Warps>, kEnc32Warps * 32,
                            kEnc32Warps * 4096 * sizeof(uint32_t)), "occupancy enc32") &&
             ctx->check(cudaFuncSetAttribute(lz4_compress_blocks_solo, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)kSoloSmemBytes), "solo smem") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->enc_solo_ctas_per_sm, lz4_compress_blocks_solo, 64,
                                                                      kSoloSmemBytes), "occupancy solo");
    }
#endif
    if (ok && ctx->enc_gtab_ctas_per_sm < kGtabCtasPerSm) {
        ctx->last_error = std::string(kGtabKernelName) + ": " + std::to_string(ctx->enc_gtab_ctas_per_sm) + " resident CTAs per SM, " +
                          std::to_string(kGtabCtasPerSm) + " planned";
        ok = false;
    }
    if (!ok || ctx->dec_ctas_per_sm < 1 || ctx->enc16s_ctas_per_sm < 1 || ctx->enc32s_ctas_per_sm < 1) {
        fprintf(stderr, "lz4b200: context creation failed: %s\n", ctx->last_error.c_str());
        lz4b200_ctx_destroy(ctx);
        return LZ4B200_CUDA_ERROR;
    }
    // The global-table encoders mark their table accesses L2::evict_last; how much of the L2 such lines may occupy is the
    // device's persisting-L2 limit (LZ4B200_L2_PERSIST_MB sets it; unset = leave the process's setting alone).
    if (const char *g = getenv("LZ4B200_L2_PERSIST_MB")) {
        int maxp = 0;
        cudaDeviceGetAttribute(&maxp, cudaDevAttrMaxPersistingL2CacheSize, device);
        const size_t bytes = std::min<size_t>((size_t)std::max(0L, atol(g)) << 20, (size_t)maxp);
        const cudaError_t e = cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, bytes);
        if (getenv("LZ4B200_DEBUG"))
            fprintf(stderr, "lz4b200: persisting L2 limit %zu of max %d bytes: %s\n", bytes, maxp, cudaGetErrorString(e));
    }
    if (const char *g = getenv("LZ4B200_ENC_G16")) ctx->enc_g16 = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_G16_CTAS")) ctx->enc_g16_ctas = std::max(1, std::min(8, atoi(g)));
#ifdef LZ4B200_AB_VARIANTS
    if (const char *g = getenv("LZ4B200_ENC_NIB")) ctx->enc_nib = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_NIB_CTAS")) ctx->enc_nib_ctas = std::max(1, std::min(8, atoi(g)));
#endif
    if (const char *g = getenv("LZ4B200_ENC_SOLO")) ctx->enc_solo = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_SOLO_SMALL_MAX")) ctx->enc_solo_small_max = (uint32_t)atoll(g);
    if (ctx->enc_solo2_ctas_per_sm < 1 && ctx->enc_solo == 2) ctx->enc_solo = 0;
    if (getenv("LZ4B200_DEBUG"))
        fprintf(stderr, "lz4b200: SMs %d, CTAs/SM: dec %d, enc16-split %d (x%d pairs), enc32-split %d (x%d pairs), solo2 %d, %s %d\n",
                ctx->sm_count, ctx->dec_ctas_per_sm, ctx->enc16s_ctas_per_sm, kEnc16Pairs, ctx->enc32s_ctas_per_sm, kEnc32Pairs,
                ctx->enc_solo2_ctas_per_sm, kGtabKernelName, ctx->enc_gtab_ctas_per_sm);
#ifdef LZ4B200_AB_VARIANTS
    if (ctx->enc_solo == 1 && ctx->enc_solo_ctas_per_sm < 1) ctx->enc_solo = 0;
    if (const char *g = getenv("LZ4B200_ENC_SINGLE_WARP")) ctx->enc_single_warp = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_GTAB")) ctx->enc_gtab = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_GTAG")) ctx->enc_gtag = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_GTAG_CTAS")) ctx->enc_gtag_ctas = std::max(1, std::min(8, atoi(g)));
    if (const char *g = getenv("LZ4B200_DEC_CTAS")) ctx->dec_ctas_override = atoi(g);
    if (const char *g = getenv("LZ4B200_DEC_BATCHED")) ctx->dec_batched = atoi(g);
    if (const char *g = getenv("LZ4B200_DEC_CONV")) ctx->dec_conv = atoi(g);
    if (const char *g = getenv("LZ4B200_THREAD_MIN")) ctx->enc_thread_min = ctx->dec_thread_min = (uint32_t)atoll(g);
    if (const char *g = getenv("LZ4B200_ENC_THREAD_MIN")) ctx->enc_thread_min = (uint32_t)atoll(g);
    if (const char *g = getenv("LZ4B200_DEC_THREAD_MIN")) ctx->dec_thread_min = (uint32_t)atoll(g);
    if (const char *g = getenv("LZ4B200_ENC_THREAD_LANES")) ctx->enc_thread_lanes = atoi(g);
    if (const char *g = getenv("LZ4B200_DEC_THREAD_LANES")) ctx->dec_thread_lanes = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_THREADS")) ctx->enc_thread_max = std::max(32, atoi(g));
    if (const char *g = getenv("LZ4B200_DEC_THREADS")) ctx->dec_thread_max = std::max(32, atoi(g));
    if (const char *g = getenv("LZ4B200_DEC_GROUP")) {
        int v = atoi(g);
        if (v == 4 || v == 8 || v == 16 || v == 32) ctx->dec_group_override = v;
    }
#else
    if (ctx->enc_solo == 1) ctx->enc_solo = 0;               // the single-thread solo kernel only exists in the A/B build
#endif
    *out = ctx;
    return LZ4B200_OK;
}

void lz4b200_ctx_destroy(lz4b200_ctx *ctx)
{
    if (!ctx) return;
    DeviceGuard guard(ctx->device);
    delete ctx;
}

void lz4b200_ctx_set_priority(lz4b200_ctx *ctx, int high)
{
    if (ctx && !ctx->pipe) ctx->high_priority = high != 0;    // takes effect when the pipeline streams are created
}

void *lz4b200_ctx_stream(lz4b200_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

const char *lz4b200_ctx_last_kernel(const lz4b200_ctx *ctx, int which)
{
    return ctx && (which == 0 || which == 1) ? ctx->last_kernel[which] : "";
}

size_t lz4b200_max_output_size(size_t n) { return 16 + 4 + (size_t)((uint64_t)n * 110 / 100); }

uint32_t lz4b200_xxh32(const uint8_t *data, size_t n, uint32_t seed) { return fw::xxh32(data, n, seed); }

void lz4b200_xxh32_reset(lz4b200_xxh32_state *st, uint32_t seed) { fw::xxh32_reset(*st, seed); }

void lz4b200_xxh32_update(lz4b200_xxh32_state *st, const uint8_t *data, size_t n) { fw::xxh32_update(*st, data, n); }

uint32_t lz4b200_xxh32_digest(const lz4b200_xxh32_state *st) { return fw::xxh32_digest(*st); }

#ifdef LZ4B200_ENC_PROFILE
// Development build only: copies the matcher's phase counters (lz4b200::EncProfSlot order) of the current device to
// out[0..16) and, if reset != 0, clears them.  Synchronises the device.
int lz4b200_enc_profile_read(uint64_t *out, int reset)
{
    if (cudaDeviceSynchronize() != cudaSuccess) return LZ4B200_CUDA_ERROR;
    if (cudaMemcpyFromSymbol(out, lz4b200::g_enc_profile, sizeof(lz4b200::g_enc_profile)) != cudaSuccess) return LZ4B200_CUDA_ERROR;
    if (reset) {
        static const unsigned long long zero[lz4b200::kEncProfSlots] = {};
        if (cudaMemcpyToSymbol(lz4b200::g_enc_profile, zero, sizeof(zero)) != cudaSuccess) return LZ4B200_CUDA_ERROR;
    }
    return LZ4B200_OK;
}
#endif

// ---- device batch entry points ----------------------------------------------------------------

lz4b200_status lz4b200_compress_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                                             const uint32_t *d_in_len, const uint8_t *d_flags, uint8_t *d_out,
                                             const uint64_t *d_out_off, const uint32_t *d_out_cap,
                                             uint32_t *d_out_len, int32_t *d_status, size_t nblocks,
                                             uint32_t max_in_len, void *stream)
{
    if (!ctx || nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_out || !d_out_off || !d_out_cap || !d_out_len || !d_status))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    BatchArgs a{d_in, d_in_off, d_in_len, d_flags, d_out, d_out_off, d_out_cap, d_out_len, d_status, nullptr,
                (uint32_t)nblocks, nullptr};
    return launch_compress(ctx, a, max_in_len, (cudaStream_t)stream);
}

lz4b200_status lz4b200_decompress_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                                               const uint32_t *d_in_len, uint8_t *d_out, const uint64_t *d_out_off,
                                               const uint32_t *d_out_cap, uint32_t *d_out_len, int32_t *d_status,
                                               uint64_t *d_err_expected, size_t nblocks, void *stream)
{
    if (!ctx || nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_out || !d_out_off || !d_out_cap || !d_out_len || !d_status))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    BatchArgs a{d_in, d_in_off, d_in_len, nullptr, d_out, d_out_off, d_out_cap, d_out_len, d_status, d_err_expected,
                (uint32_t)nblocks, nullptr};
    return launch_decompress(ctx, a, (cudaStream_t)stream);
}

// Device-pointer batches with an external dictionary shared by every block (d_dict: the LAST min(len, 65536)
// bytes of the dictionary, already on the device; compress drops dictionaries of <= 3 bytes like the reference).
lz4b200_status lz4b200_compress_batch_device_with_dict(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                                                       const uint32_t *d_in_len, const uint8_t *d_dict, size_t dict_len,
                                                       uint8_t *d_out, const uint64_t *d_out_off,
                                                       const uint32_t *d_out_cap, uint32_t *d_out_len,
                                                       int32_t *d_status, size_t nblocks, uint32_t max_in_len,
                                                       void *stream)
{
    if (!ctx || nblocks > 0xffffffffull || (!d_dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_out || !d_out_off || !d_out_cap || !d_out_len || !d_status))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    BatchArgs a{d_in, d_in_off, d_in_len, nullptr, d_out, d_out_off, d_out_cap, d_out_len, d_status, nullptr,
                (uint32_t)nblocks, nullptr};
    set_dict(a, d_dict, dict_len, true);
    return launch_compress(ctx, a, max_in_len, (cudaStream_t)stream);
}

lz4b200_status lz4b200_decompress_batch_device_with_dict(lz4b200_ctx *ctx, const uint8_t *d_in,
                                                         const uint64_t *d_in_off, const uint32_t *d_in_len,
                                                         const uint8_t *d_dict, size_t dict_len, uint8_t *d_out,
                                                         const uint64_t *d_out_off, const uint32_t *d_out_cap,
                                                         uint32_t *d_out_len, int32_t *d_status,
                                                         uint64_t *d_err_expected, size_t nblocks, void *stream)
{
    if (!ctx || nblocks > 0xffffffffull || (!d_dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_out || !d_out_off || !d_out_cap || !d_out_len || !d_status))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    BatchArgs a{d_in, d_in_off, d_in_len, nullptr, d_out, d_out_off, d_out_cap, d_out_len, d_status, d_err_expected,
                (uint32_t)nblocks, nullptr};
    set_dict(a, d_dict, dict_len, false);
    return launch_decompress(ctx, a, (cudaStream_t)stream);
}

}  // extern "C"

namespace {

// lz4b200_compress_prepend_size_batch_device(_with_dict): compress every block into a slot of max_output_size(max_in_len)
// bytes with the block API's launch, scan the record sizes into rec_off, then write each record that fits at its offset.
lz4b200_status compress_prepend_size_batch(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                                           const uint32_t *d_in_len, size_t nblocks, uint32_t max_in_len,
                                           const uint8_t *d_dict, size_t dict_len, uint8_t *d_out, size_t out_cap,
                                           uint64_t *d_rec_off, int32_t *d_status, void *stream)
{
    if (!ctx || !d_rec_off || nblocks > 0xffffffffull || (!d_dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_status || (!d_out && out_cap))) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (nblocks == 0) {
        CTX_CUDA(ctx, cudaMemsetAsync(d_rec_off, 0, 8, s));
        return LZ4B200_OK;
    }
    const uint32_t n = (uint32_t)nblocks, grid = (n + 127) / 128;
    const uint32_t slot = (uint32_t)std::min<size_t>(lz4b200_max_output_size(max_in_len), 0xffffffffu);
    CTX_CUDA(ctx, ctx->d_slots.reserve((size_t)n * slot + 16));
    CTX_CUDA(ctx, ctx->d_in_len.reserve(n)); CTX_CUDA(ctx, ctx->d_out_off.reserve(n));
    CTX_CUDA(ctx, ctx->d_out_cap.reserve(n)); CTX_CUDA(ctx, ctx->d_out_len.reserve(n));
    CTX_CUDA(ctx, ctx->d_seg_size.reserve(n)); CTX_CUDA(ctx, ctx->d_gdst.reserve(n));
    CTX_CUDA(ctx, ctx->d_payload_len.reserve(n));
    prepend_desc_kernel<<<grid, 128, 0, s>>>(d_in_len, n, max_in_len, slot, ctx->d_in_len.p, ctx->d_out_off.p,
                                             ctx->d_out_cap.p);
    CTX_CUDA(ctx, cudaGetLastError());
    BatchArgs a{d_in, d_in_off, ctx->d_in_len.p, nullptr, ctx->d_slots.p, ctx->d_out_off.p, ctx->d_out_cap.p,
                ctx->d_out_len.p, d_status, nullptr, n, nullptr};
    set_dict(a, d_dict, dict_len, true);
    const lz4b200_status st = launch_compress(ctx, a, max_in_len, s);
    if (st != LZ4B200_OK) return st;
    prepend_size_kernel<<<grid, 128, 0, s>>>(ctx->d_out_len.p, d_status, n, ctx->d_seg_size.p);
    CTX_CUDA(ctx, cudaGetLastError());
    scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_seg_size.p, d_rec_off, n);
    CTX_CUDA(ctx, cudaGetLastError());
    prepend_place_kernel<<<grid, 128, 0, s>>>(d_in_len, ctx->d_out_len.p, d_rec_off, n, out_cap, d_out, d_status,
                                              ctx->d_gdst.p, ctx->d_payload_len.p);
    CTX_CUDA(ctx, cudaGetLastError());
    GatherArgs g{ctx->d_slots.p, nullptr, ctx->d_out_off.p, nullptr, ctx->d_payload_len.p, nullptr, nullptr, nullptr,
                 d_out, ctx->d_gdst.p, n};
    gather_segments_kernel<<<std::min<uint32_t>(std::max<uint32_t>(n, (uint32_t)ctx->sm_count * 2),
                                                (uint32_t)ctx->sm_count * 8), 256, 0, s>>>(g);
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}

// lz4b200_decompress_size_prepended_batch_device(_with_dict): the length words give the output layout on the device, so
// every record decodes in place into d_out with the block API's launch, and nothing returns to the host.
lz4b200_status decompress_size_prepended_batch(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_rec_off,
                                               const uint32_t *d_rec_len, size_t nrec, const uint8_t *d_dict,
                                               size_t dict_len, uint8_t *d_out, size_t out_cap, uint64_t *d_out_off,
                                               uint32_t *d_out_len, int32_t *d_status, uint64_t *d_err_expected,
                                               void *stream)
{
    if (!ctx || !d_out_off || nrec > 0xffffffffull || (!d_dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    if (nrec && (!d_in || !d_rec_off || !d_rec_len || !d_out_len || !d_status || (!d_out && out_cap)))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (nrec == 0) {
        CTX_CUDA(ctx, cudaMemsetAsync(d_out_off, 0, 8, s));
        return LZ4B200_OK;
    }
    const uint32_t n = (uint32_t)nrec, grid = (n + 127) / 128;
    CTX_CUDA(ctx, ctx->d_seg_size.reserve(n)); CTX_CUDA(ctx, ctx->d_in_off.reserve(n));
    CTX_CUDA(ctx, ctx->d_in_len.reserve(n)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(n));
    CTX_CUDA(ctx, ctx->d_pick.reserve(n));
    prepended_size_kernel<<<grid, 128, 0, s>>>(d_in, d_rec_off, d_rec_len, n, ctx->d_seg_size.p);
    CTX_CUDA(ctx, cudaGetLastError());
    scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_seg_size.p, d_out_off, n);
    CTX_CUDA(ctx, cudaGetLastError());
    prepended_args_kernel<<<grid, 128, 0, s>>>(d_rec_off, d_rec_len, ctx->d_seg_size.p, d_out_off, n, out_cap,
                                               ctx->d_in_off.p, ctx->d_in_len.p, ctx->d_out_cap.p, ctx->d_pick.p);
    CTX_CUDA(ctx, cudaGetLastError());
    BatchArgs a{d_in, ctx->d_in_off.p, ctx->d_in_len.p, nullptr, d_out, d_out_off, ctx->d_out_cap.p, d_out_len, d_status,
                d_err_expected, n, nullptr};
    set_dict(a, d_dict, dict_len, false);
    const lz4b200_status st = launch_decompress(ctx, a, s);
    if (st != LZ4B200_OK) return st;
    prepended_status_kernel<<<grid, 128, 0, s>>>(ctx->d_pick.p, n, d_status);
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}

}  // namespace

extern "C" {

// ---- many size-prepended blocks, device pointers --------------------------------------------------------------------

lz4b200_status lz4b200_compress_prepend_size_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                                                          const uint32_t *d_in_len, size_t nblocks, uint32_t max_in_len,
                                                          uint8_t *d_out, size_t out_cap, uint64_t *d_rec_off,
                                                          int32_t *d_status, void *stream)
{
    return compress_prepend_size_batch(ctx, d_in, d_in_off, d_in_len, nblocks, max_in_len, nullptr, 0, d_out, out_cap,
                                       d_rec_off, d_status, stream);
}

lz4b200_status lz4b200_compress_prepend_size_batch_device_with_dict(lz4b200_ctx *ctx, const uint8_t *d_in,
                                                                    const uint64_t *d_in_off, const uint32_t *d_in_len,
                                                                    size_t nblocks, uint32_t max_in_len,
                                                                    const uint8_t *d_dict, size_t dict_len,
                                                                    uint8_t *d_out, size_t out_cap, uint64_t *d_rec_off,
                                                                    int32_t *d_status, void *stream)
{
    return compress_prepend_size_batch(ctx, d_in, d_in_off, d_in_len, nblocks, max_in_len, d_dict, dict_len, d_out,
                                       out_cap, d_rec_off, d_status, stream);
}

lz4b200_status lz4b200_decompress_size_prepended_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in,
                                                              const uint64_t *d_rec_off, const uint32_t *d_rec_len,
                                                              size_t nrec, uint8_t *d_out, size_t out_cap,
                                                              uint64_t *d_out_off, uint32_t *d_out_len, int32_t *d_status,
                                                              uint64_t *d_err_expected, void *stream)
{
    return decompress_size_prepended_batch(ctx, d_in, d_rec_off, d_rec_len, nrec, nullptr, 0, d_out, out_cap, d_out_off,
                                           d_out_len, d_status, d_err_expected, stream);
}

lz4b200_status lz4b200_decompress_size_prepended_batch_device_with_dict(lz4b200_ctx *ctx, const uint8_t *d_in,
                                                                        const uint64_t *d_rec_off,
                                                                        const uint32_t *d_rec_len, size_t nrec,
                                                                        const uint8_t *d_dict, size_t dict_len,
                                                                        uint8_t *d_out, size_t out_cap,
                                                                        uint64_t *d_out_off, uint32_t *d_out_len,
                                                                        int32_t *d_status, uint64_t *d_err_expected,
                                                                        void *stream)
{
    return decompress_size_prepended_batch(ctx, d_in, d_rec_off, d_rec_len, nrec, d_dict, dict_len, d_out, out_cap,
                                           d_out_off, d_out_len, d_status, d_err_expected, stream);
}

// ---- host batch entry points --------------------------------------------------------------------
// Both calls are chunked software pipelines over kLanes streams: while chunk c runs its kernel, chunk
// c+1's input crosses PCIe host->device and chunk c-1's result crosses device->host (full duplex), so
// a large batch runs at max(PCIe, kernel) instead of their sum.

}  // extern "C"

namespace {

// Lanes in flight.  A compress chunk occupies its lane for H2D + kernel (at least one block's serial chain, several ms)
// + the size read-back + D2H, so a few lanes cap the call whatever the kernel does; eight lanes leave the kernel / PCIe as
// the bound.  LZ4B200_LANES overrides.
static int lanes_in_use()
{
    static const int v = [] { const char *e = getenv("LZ4B200_LANES"); int k = e ? atoi(e) : 8; return k < 1 ? 1 : (k > kMaxLanes ? kMaxLanes : k); }();
    return v;
}
// decompress: a chunk's kernel lasts at least one block's serial chain (about a millisecond for 64 KiB of JSON) however
// few blocks it holds, so chunks must be big enough for that to hide behind the chunk's own D2H copy
constexpr uint64_t kChunkBytesDefault = 128ull << 20;
// compress: a 64 KiB block is one serial chain of several ms whatever the batch size, so a chunk must hold enough blocks
// (2048) for two chunks in flight to fill the GPU
constexpr uint64_t kCompressChunkBytesDefault = 128ull << 20;

uint64_t env_mib(const char *name, uint64_t dflt)         // tuning aid: chunk sizes in MiB
{
    const char *v = getenv(name);
    const long m = v ? atol(v) : 0;
    return m > 0 ? (uint64_t)m << 20 : dflt;
}

lz4b200_status pipeline_init(lz4b200_ctx *ctx, Pipeline &p)
{
    if (p.ready) return LZ4B200_OK;
    // LZ4B200_STREAM_PRIORITY=high: this context's kernels get the SM slots first when another context (e.g. a
    // compress pipeline running next to a decompress pipeline) keeps the GPU full
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);
    const int prio = ctx->high_priority ? hi : 0;
    for (Lane &l : p.lane) {
        if (!l.stream) CTX_CUDA(ctx, cudaStreamCreateWithPriority(&l.stream, cudaStreamNonBlocking, prio));
        if (!l.sizes_ready) CTX_CUDA(ctx, cudaEventCreateWithFlags(&l.sizes_ready, cudaEventDisableTiming));
    }
    if (!p.desc_ready) CTX_CUDA(ctx, cudaEventCreateWithFlags(&p.desc_ready, cudaEventDisableTiming));
    if (!p.d_tickets.p) CTX_CUDA(ctx, p.d_tickets.resize(kMaxLanes * 8));
    CTX_CUDA(ctx, cudaMemset(p.d_tickets.p, 0, kMaxLanes * 8 * sizeof(uint32_t)));
    ctx->pipe_tickets = p.d_tickets.p;
    p.ready = true;
    return LZ4B200_OK;
}

Pipeline &ctx_pipeline(lz4b200_ctx *ctx)
{
    if (!ctx->pipe) ctx->pipe = std::make_unique<Pipeline>();
    return *ctx->pipe;
}

struct Chunk { uint32_t b0, b1; uint64_t in_lo, in_hi, a, b; };   // a/b: slot bytes (compress) or out_lo/out_hi (decompress)

}  // namespace

static lz4b200_status compress_batch_host_impl(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                               const uint32_t *in_len, const uint8_t *flags, const uint8_t *dict,
                                               size_t dict_len, uint8_t *out, size_t out_cap_total, uint64_t *out_off,
                                               uint32_t *out_len, int32_t *status, size_t nblocks)
{
    if (!ctx || nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks == 0) return LZ4B200_OK;
    if (!in || !in_off || !in_len || !out || !out_off || !out_len || !status) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    Pipeline &pl = ctx_pipeline(ctx);
    const int kLanes = lanes_in_use();
    lz4b200_status st = pipeline_init(ctx, pl);
    if (st != LZ4B200_OK) return st;
    const uint32_t nb = (uint32_t)nblocks;

    // ---- plan: chunks of ~kCompressChunkBytes input, descriptors relative to each chunk's buffers ------
    static const uint64_t kCompressChunkBytes = env_mib("LZ4B200_ENC_CHUNK_MB", kCompressChunkBytesDefault);
    std::vector<Chunk> chunks;
    std::vector<uint64_t> h_in_off(nb), h_slot_off(nb);
    std::vector<uint32_t> h_cap(nb);
    uint32_t max_len = 0;
    for (uint32_t b = 0; b < nb;) {
        Chunk c{b, b, ~0ull, 0, 0, 0};
        uint64_t bytes = 0;
        // ramp: the first chunks are small (32, 64, ... MiB) so the first kernel starts after a short copy.  (Shrinking the
        // LAST chunks as well — so that less work waits behind the last copy — was measured slower: the extra chunks'
        // read-back / pack / D2H round trips cost more than the shorter tail saves.)
        const uint64_t limit = std::min<uint64_t>(kCompressChunkBytes, (32ull << 20) << std::min<size_t>(chunks.size(), 8));
        while (c.b1 < nb && (c.b1 == c.b0 || bytes + in_len[c.b1] <= limit)) {
            const uint32_t k = c.b1++;
            c.in_lo = std::min<uint64_t>(c.in_lo, in_off[k]);
            c.in_hi = std::max<uint64_t>(c.in_hi, in_off[k] + in_len[k]);
            bytes += in_len[k];
            max_len = std::max(max_len, in_len[k]);
            const size_t m = lz4b200_max_output_size(in_len[k]);
            if (m > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
            h_cap[k] = (uint32_t)m;
            h_slot_off[k] = c.a;
            c.a += (m + 15) & ~size_t(15);
        }
        for (uint32_t k = c.b0; k < c.b1; k++) h_in_off[k] = in_off[k] - c.in_lo;
        chunks.push_back(c);
        b = c.b1;
    }
    const uint32_t nch = (uint32_t)chunks.size();
    CTX_CUDA(ctx, ctx->d_in_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_in_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_status.reserve(nb));
    CTX_CUDA(ctx, ctx->d_seg_off.reserve(nb + nch));
    if (flags) CTX_CUDA(ctx, ctx->d_flags.reserve(nb));
    CTX_CUDA(ctx, pl.h_seg.reserve((size_t)nb + nch));
    CTX_CUDA(ctx, pl.h_status.reserve(nb));

    cudaStream_t s0 = pl.lane[0].stream;
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_off.p, h_in_off.data(), nb * 8, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_len.p, in_len, nb * 4, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_off.p, h_slot_off.data(), nb * 8, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_cap.p, h_cap.data(), nb * 4, cudaMemcpyHostToDevice, s0));
    if (flags) CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_flags.p, flags, nb, cudaMemcpyHostToDevice, s0));
    normalize_dict(dict, dict_len, true);
    if (dict_len) {
        CTX_CUDA(ctx, ctx->d_dict.reserve(dict_len + 16));
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_dict.p, dict, dict_len, cudaMemcpyHostToDevice, s0));
    }
    CTX_CUDA(ctx, cudaEventRecord(pl.desc_ready, s0));
    CTX_CUDA(ctx, cudaStreamSynchronize(s0));            // the host vectors above may go out of scope before use otherwise

    auto phase1 = [&](uint32_t ci) -> lz4b200_status {  // H2D + kernel + scan + sizes D2H
        const Chunk &c = chunks[ci];
        Lane &ln = pl.lane[ci % kLanes];
        const uint32_t n = c.b1 - c.b0;
        CTX_CUDA(ctx, ln.in.reserve(c.in_hi - c.in_lo + 16));
        CTX_CUDA(ctx, ln.slots.reserve(c.a + 16));
        CTX_CUDA(ctx, cudaStreamWaitEvent(ln.stream, pl.desc_ready, 0));
        CTX_CUDA(ctx, cudaMemcpyAsync(ln.in.p, in + c.in_lo, c.in_hi - c.in_lo, cudaMemcpyHostToDevice, ln.stream));
        BatchArgs a{ln.in.p, ctx->d_in_off.p + c.b0, ctx->d_in_len.p + c.b0, flags ? ctx->d_flags.p + c.b0 : nullptr,
                    ln.slots.p, ctx->d_out_off.p + c.b0, ctx->d_out_cap.p + c.b0, ctx->d_out_len.p + c.b0,
                    ctx->d_status.p + c.b0, nullptr, n, nullptr};
        if (dict_len) { a.dict = ctx->d_dict.p; a.dict_len = (uint32_t)dict_len; }
        lz4b200_status r = launch_compress(ctx, a, max_len, ln.stream, pl.d_tickets.p + 8 * (ci % kLanes));
        if (r != LZ4B200_OK) return r;
        scan_sizes_kernel<<<1, 1024, 0, ln.stream>>>(ctx->d_out_len.p + c.b0, ctx->d_seg_off.p + c.b0 + ci, n);
        CTX_CUDA(ctx, cudaGetLastError());
        CTX_CUDA(ctx, cudaMemcpyAsync(pl.h_seg.p + c.b0 + ci, ctx->d_seg_off.p + c.b0 + ci, (n + 1) * 8,
                                      cudaMemcpyDeviceToHost, ln.stream));
        CTX_CUDA(ctx, cudaEventRecord(ln.sizes_ready, ln.stream));
        return LZ4B200_OK;
    };

    for (uint32_t ci = 0; ci < nch && ci < (uint32_t)kLanes; ci++) {
        st = phase1(ci);
        if (st != LZ4B200_OK) return st;
    }
    uint64_t out_base = 0;
    lz4b200_status result = LZ4B200_OK;
    for (uint32_t ci = 0; ci < nch; ci++) {
        const Chunk &c = chunks[ci];
        Lane &ln = pl.lane[ci % kLanes];
        const uint32_t n = c.b1 - c.b0;
        CTX_CUDA(ctx, cudaEventSynchronize(ln.sizes_ready));
        const uint64_t *seg = pl.h_seg.p + c.b0 + ci;
        const uint64_t total = seg[n];
        for (uint32_t k = 0; k < n; k++) {
            out_off[c.b0 + k] = out_base + seg[k];
            out_len[c.b0 + k] = (uint32_t)(seg[k + 1] - seg[k]);
        }
        if (out_base + total > out_cap_total) { result = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL; break; }
        if (total) {
            CTX_CUDA(ctx, ln.out.reserve(total + 16));
            GatherArgs g{ln.slots.p, nullptr, ctx->d_out_off.p + c.b0, nullptr, ctx->d_out_len.p + c.b0, nullptr, nullptr,
                         nullptr, ln.out.p, ctx->d_seg_off.p + c.b0 + ci, n};
            gather_segments_kernel<<<std::min<uint32_t>(n, (uint32_t)ctx->sm_count * 8), 256, 0, ln.stream>>>(g);
            CTX_CUDA(ctx, cudaGetLastError());
            CTX_CUDA(ctx, cudaMemcpyAsync(out + out_base, ln.out.p, total, cudaMemcpyDeviceToHost, ln.stream));
        }
        out_base += total;
        if (ci + kLanes < nch) {
            st = phase1(ci + kLanes);
            if (st != LZ4B200_OK) return st;
        }
    }
    for (int i = 0; i < kLanes; i++) CTX_CUDA(ctx, cudaStreamSynchronize(pl.lane[i].stream));
    if (result != LZ4B200_OK) return result;
    CTX_CUDA(ctx, cudaMemcpyAsync(pl.h_status.p, ctx->d_status.p, nb * 4, cudaMemcpyDeviceToHost, s0));
    CTX_CUDA(ctx, cudaStreamSynchronize(s0));
    memcpy(status, pl.h_status.p, nb * 4);
    return LZ4B200_OK;
}

static lz4b200_status decompress_batch_host_impl(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                                 const uint32_t *in_len, const uint8_t *dict, size_t dict_len,
                                                 uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
                                                 uint32_t *out_len, int32_t *status, uint64_t *err_expected,
                                                 size_t nblocks)
{
    if (!ctx || nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks == 0) return LZ4B200_OK;
    if (!in || !in_off || !in_len || !out || !out_off || !out_cap || !out_len || !status)
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    Pipeline &pl = ctx_pipeline(ctx);
    const int kLanes = lanes_in_use();
    lz4b200_status st = pipeline_init(ctx, pl);
    if (st != LZ4B200_OK) return st;
    const uint32_t nb = (uint32_t)nblocks;

    static const uint64_t kChunkBytes = env_mib("LZ4B200_DEC_CHUNK_MB", kChunkBytesDefault);
    std::vector<Chunk> chunks;
    std::vector<uint8_t> contiguous;
    std::vector<uint64_t> h_in_off(nb), h_out_off(nb);
    for (uint32_t b = 0; b < nb;) {
        Chunk c{b, b, ~0ull, 0, ~0ull, 0};
        uint64_t bytes = 0;
        bool contig = true;
        const uint64_t limit = std::min<uint64_t>(kChunkBytes, (32ull << 20) << std::min<size_t>(chunks.size(), 8));
        while (c.b1 < nb && (c.b1 == c.b0 || bytes + out_cap[c.b1] <= limit)) {
            const uint32_t k = c.b1++;
            c.in_lo = std::min<uint64_t>(c.in_lo, in_off[k]); c.in_hi = std::max<uint64_t>(c.in_hi, in_off[k] + in_len[k]);
            c.a = std::min<uint64_t>(c.a, out_off[k]); c.b = std::max<uint64_t>(c.b, out_off[k] + out_cap[k]);
            if (k > c.b0 && out_off[k] != out_off[k - 1] + out_cap[k - 1]) contig = false;
            bytes += out_cap[k];
        }
        for (uint32_t k = c.b0; k < c.b1; k++) { h_in_off[k] = in_off[k] - c.in_lo; h_out_off[k] = out_off[k] - c.a; }
        chunks.push_back(c);
        contiguous.push_back(contig ? 1 : 0);
        b = c.b1;
    }
    const uint32_t nch = (uint32_t)chunks.size();
    CTX_CUDA(ctx, ctx->d_in_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_in_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_status.reserve(nb));
    CTX_CUDA(ctx, ctx->d_expected.reserve(nb));
    CTX_CUDA(ctx, pl.h_seg.reserve((size_t)nb));
    CTX_CUDA(ctx, pl.h_status.reserve((size_t)nb * 2));
    cudaStream_t s0 = pl.lane[0].stream;
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_off.p, h_in_off.data(), nb * 8, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_len.p, in_len, nb * 4, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_off.p, h_out_off.data(), nb * 8, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_cap.p, out_cap, nb * 4, cudaMemcpyHostToDevice, s0));
    normalize_dict(dict, dict_len, false);
    if (dict_len) {
        CTX_CUDA(ctx, ctx->d_dict.reserve(dict_len + 16));
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_dict.p, dict, dict_len, cudaMemcpyHostToDevice, s0));
    }
    CTX_CUDA(ctx, cudaEventRecord(pl.desc_ready, s0));
    CTX_CUDA(ctx, cudaStreamSynchronize(s0));

    for (uint32_t ci = 0; ci < nch; ci++) {
        const Chunk &c = chunks[ci];
        Lane &ln = pl.lane[ci % kLanes];
        const uint32_t n = c.b1 - c.b0;
        CTX_CUDA(ctx, ln.in.reserve(c.in_hi - c.in_lo + 16));
        CTX_CUDA(ctx, ln.out.reserve(c.b - c.a + 16));
        CTX_CUDA(ctx, cudaStreamWaitEvent(ln.stream, pl.desc_ready, 0));
        CTX_CUDA(ctx, cudaMemcpyAsync(ln.in.p, in + c.in_lo, c.in_hi - c.in_lo, cudaMemcpyHostToDevice, ln.stream));
        // The whole capacity region of every slot travels back (the decoded sizes are only known after the kernel), so
        // what lies past a block's decoded length must not be whatever an earlier call left in this staging buffer.
        CTX_CUDA(ctx, cudaMemsetAsync(ln.out.p, 0, c.b - c.a, ln.stream));
        BatchArgs a{ln.in.p, ctx->d_in_off.p + c.b0, ctx->d_in_len.p + c.b0, nullptr, ln.out.p, ctx->d_out_off.p + c.b0,
                    ctx->d_out_cap.p + c.b0, ctx->d_out_len.p + c.b0, ctx->d_status.p + c.b0, ctx->d_expected.p + c.b0, n,
                    nullptr};
        if (dict_len) { a.dict = ctx->d_dict.p; a.dict_len = (uint32_t)dict_len; }
        st = launch_decompress(ctx, a, ln.stream, pl.d_tickets.p + 8 * (ci % kLanes));
        if (st != LZ4B200_OK) return st;
        if (contiguous[ci]) {
            CTX_CUDA(ctx, cudaMemcpyAsync(out + c.a, ln.out.p, c.b - c.a, cudaMemcpyDeviceToHost, ln.stream));
        } else {
            for (uint32_t k = c.b0; k < c.b1; k++)
                if (out_cap[k])
                    CTX_CUDA(ctx, cudaMemcpyAsync(out + out_off[k], ln.out.p + h_out_off[k], out_cap[k],
                                                  cudaMemcpyDeviceToHost, ln.stream));
        }
    }
    for (int i = 0; i < kLanes; i++) CTX_CUDA(ctx, cudaStreamSynchronize(pl.lane[i].stream));
    uint32_t *h_len = reinterpret_cast<uint32_t *>(pl.h_status.p + nb);
    CTX_CUDA(ctx, cudaMemcpyAsync(pl.h_status.p, ctx->d_status.p, nb * 4, cudaMemcpyDeviceToHost, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(h_len, ctx->d_out_len.p, nb * 4, cudaMemcpyDeviceToHost, s0));
    if (err_expected)
        CTX_CUDA(ctx, cudaMemcpyAsync(pl.h_seg.p, ctx->d_expected.p, nb * 8, cudaMemcpyDeviceToHost, s0));
    CTX_CUDA(ctx, cudaStreamSynchronize(s0));
    memcpy(status, pl.h_status.p, nb * 4);
    memcpy(out_len, h_len, nb * 4);
    if (err_expected) memcpy(err_expected, pl.h_seg.p, nb * 8);
    return LZ4B200_OK;
}

extern "C" {

lz4b200_status lz4b200_compress_batch_host(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                           const uint32_t *in_len, const uint8_t *flags, uint8_t *out,
                                           size_t out_cap_total, uint64_t *out_off, uint32_t *out_len,
                                           int32_t *status, size_t nblocks)
{
    return compress_batch_host_impl(ctx, in, in_off, in_len, flags, nullptr, 0, out, out_cap_total, out_off, out_len,
                                    status, nblocks);
}

lz4b200_status lz4b200_decompress_batch_host(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                             const uint32_t *in_len, uint8_t *out, const uint64_t *out_off,
                                             const uint32_t *out_cap, uint32_t *out_len, int32_t *status,
                                             uint64_t *err_expected, size_t nblocks)
{
    return decompress_batch_host_impl(ctx, in, in_off, in_len, nullptr, 0, out, out_off, out_cap, out_len, status,
                                      err_expected, nblocks);
}

lz4b200_status lz4b200_compress_batch_host_with_dict(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                                     const uint32_t *in_len, const uint8_t *dict, size_t dict_len,
                                                     uint8_t *out, size_t out_cap_total, uint64_t *out_off,
                                                     uint32_t *out_len, int32_t *status, size_t nblocks)
{
    return compress_batch_host_impl(ctx, in, in_off, in_len, nullptr, dict, dict_len, out, out_cap_total, out_off,
                                    out_len, status, nblocks);
}

lz4b200_status lz4b200_decompress_batch_host_with_dict(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                                       const uint32_t *in_len, const uint8_t *dict, size_t dict_len,
                                                       uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
                                                       uint32_t *out_len, int32_t *status, uint64_t *err_expected,
                                                       size_t nblocks)
{
    return decompress_batch_host_impl(ctx, in, in_off, in_len, dict, dict_len, out, out_off, out_cap, out_len, status,
                                      err_expected, nblocks);
}

// ---- single-block host entry points -----------------------------------------------------------

lz4b200_status lz4b200_compress_into(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                     size_t *written)
{
    if (!ctx || !written || (!in && n) || n > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (cap < lz4b200_max_output_size(n)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;     // compress.rs:338-340
    uint64_t in_off = 0, out_off = 0;
    uint32_t in_len = (uint32_t)n, out_len = 0;
    int32_t status = 0;
    static const uint8_t zero = 0;
    lz4b200_status st = lz4b200_compress_batch_host(ctx, n ? in : &zero, &in_off, &in_len, nullptr, out, cap, &out_off,
                                                    &out_len, &status, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) return (lz4b200_status)status;
    *written = out_len;
    return LZ4B200_OK;
}

lz4b200_status lz4b200_compress_prepend_size(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                             size_t *written)
{
    if (!written) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (cap < 4) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    wr32(out, (uint32_t)n);                                                              // compress.rs:633/649
    size_t w = 0;
    lz4b200_status st = lz4b200_compress_into(ctx, in, n, out + 4, cap - 4, &w);
    if (st == LZ4B200_OK) *written = w + 4;
    return st;
}

lz4b200_status lz4b200_decompress_into(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                       size_t *written, size_t *err_expected, size_t *err_actual)
{
    if (!ctx || !written || n > 0xffffffffull || cap > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (err_expected) *err_expected = 0;
    if (err_actual) *err_actual = 0;
    if (n == 0) return LZ4B200_DEC_EXPECTED_ANOTHER_BYTE;                                // decompress.rs:207-209
    uint64_t in_off = 0, out_off = 0, expected = 0;
    uint32_t in_len = (uint32_t)n, out_cap = (uint32_t)cap, out_len = 0;
    int32_t status = 0;
    uint8_t dummy = 0;
    lz4b200_status st = lz4b200_decompress_batch_host(ctx, in, &in_off, &in_len, cap ? out : &dummy, &out_off, &out_cap,
                                                      &out_len, &status, &expected, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) {
        if (status == LZ4B200_DEC_OUTPUT_TOO_SMALL) {
            if (err_expected) *err_expected = (size_t)expected;
            if (err_actual) *err_actual = cap;
        }
        return (lz4b200_status)status;
    }
    *written = out_len;
    return LZ4B200_OK;
}

// ---- external dictionary (compress.rs:610-616, 685-693; decompress.rs:462-468, 478-528) ------------------

lz4b200_status lz4b200_compress_into_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n, const uint8_t *dict,
                                               size_t dict_len, uint8_t *out, size_t cap, size_t *written)
{
    if (!ctx || !written || (!in && n) || n > 0xffffffffull || (!dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (cap < lz4b200_max_output_size(n)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;     // compress.rs:338-340
    uint64_t in_off = 0, out_off = 0;
    uint32_t in_len = (uint32_t)n, out_len = 0;
    int32_t status = 0;
    static const uint8_t zero = 0;
    lz4b200_status st = compress_batch_host_impl(ctx, n ? in : &zero, &in_off, &in_len, nullptr, dict, dict_len, out, cap,
                                                 &out_off, &out_len, &status, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) return (lz4b200_status)status;
    *written = out_len;
    return LZ4B200_OK;
}

// block::compress_into_with_table (compress.rs:744-766).  The reusable CompressTable only decides which table
// layout / hash the parse uses: Small = u16 entries + 4-byte hash (inputs < 65 535 bytes), Large = u32 entries +
// 5-byte hash for any size; a Small table handed an input >= 65 535 bytes is upgraded to Large and stays Large.
// *table_kind carries that state (LZ4B200_TABLE_SMALL / LZ4B200_TABLE_LARGE); the table's memory lives on the GPU.
lz4b200_status lz4b200_compress_into_with_table(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                                size_t *written, int *table_kind)
{
    if (!ctx || !written || !table_kind || (!in && n) || n > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (*table_kind != LZ4B200_TABLE_SMALL && *table_kind != LZ4B200_TABLE_LARGE) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (n >= 65535 && *table_kind == LZ4B200_TABLE_SMALL) *table_kind = LZ4B200_TABLE_LARGE;      // compress.rs:750-752
    if (cap < lz4b200_max_output_size(n)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;                // compress.rs:338-340
    uint64_t in_off = 0, out_off = 0;
    uint32_t in_len = (uint32_t)n, out_len = 0;
    int32_t status = 0;
    const uint8_t flag = *table_kind == LZ4B200_TABLE_LARGE ? (uint8_t)LZ4B200_BLOCK_HASH5_ALWAYS : (uint8_t)0;
    static const uint8_t zero = 0;
    lz4b200_status st = compress_batch_host_impl(ctx, n ? in : &zero, &in_off, &in_len, &flag, nullptr, 0, out, cap,
                                                 &out_off, &out_len, &status, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) return (lz4b200_status)status;
    *written = out_len;
    return LZ4B200_OK;
}

lz4b200_status lz4b200_compress_prepend_size_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                       const uint8_t *dict, size_t dict_len, uint8_t *out, size_t cap,
                                                       size_t *written)
{
    if (!written) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (cap < 4) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    wr32(out, (uint32_t)n);
    size_t w = 0;
    lz4b200_status st = lz4b200_compress_into_with_dict(ctx, in, n, dict, dict_len, out + 4, cap - 4, &w);
    if (st == LZ4B200_OK) *written = w + 4;
    return st;
}

lz4b200_status lz4b200_decompress_into_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n, const uint8_t *dict,
                                                 size_t dict_len, uint8_t *out, size_t cap, size_t *written,
                                                 size_t *err_expected, size_t *err_actual)
{
    if (!ctx || !written || n > 0xffffffffull || cap > 0xffffffffull || (!dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (err_expected) *err_expected = 0;
    if (err_actual) *err_actual = 0;
    if (n == 0) return LZ4B200_DEC_EXPECTED_ANOTHER_BYTE;                                // decompress.rs:207-209
    uint64_t in_off = 0, out_off = 0, expected = 0;
    uint32_t in_len = (uint32_t)n, out_cap = (uint32_t)cap, out_len = 0;
    int32_t status = 0;
    uint8_t dummy = 0;
    lz4b200_status st = decompress_batch_host_impl(ctx, in, &in_off, &in_len, dict, dict_len, cap ? out : &dummy, &out_off,
                                                   &out_cap, &out_len, &status, &expected, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) {
        if (status == LZ4B200_DEC_OUTPUT_TOO_SMALL) {
            if (err_expected) *err_expected = (size_t)expected;
            if (err_actual) *err_actual = cap;
        }
        return (lz4b200_status)status;
    }
    *written = out_len;
    return LZ4B200_OK;
}

lz4b200_status lz4b200_decompress_size_prepended_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                           const uint8_t *dict, size_t dict_len, uint8_t *out,
                                                           size_t cap, size_t *written, size_t *err_expected,
                                                           size_t *err_actual)
{
    size_t want = 0;
    if (written) *written = 0;
    lz4b200_status st = lz4b200_uncompressed_size(in, n, &want);
    if (st != LZ4B200_OK) return st;
    if (cap < want) return LZ4B200_INVALID_ARGUMENT;
    return lz4b200_decompress_into_with_dict(ctx, in + 4, n - 4, dict, dict_len, out, want, written, err_expected,
                                             err_actual);
}

lz4b200_status lz4b200_uncompressed_size(const uint8_t *in, size_t n, size_t *size)
{
    if (!size) return LZ4B200_INVALID_ARGUMENT;
    if (n < 4) return LZ4B200_DEC_EXPECTED_ANOTHER_BYTE;                                 // block/mod.rs:151-157
    *size = rd32(in);
    return LZ4B200_OK;
}

lz4b200_status lz4b200_decompress_size_prepended(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out,
                                                 size_t cap, size_t *written, size_t *err_expected,
                                                 size_t *err_actual)
{
    size_t want = 0;
    if (written) *written = 0;
    lz4b200_status st = lz4b200_uncompressed_size(in, n, &want);
    if (st != LZ4B200_OK) return st;
    if (cap < want) return LZ4B200_INVALID_ARGUMENT;
    return lz4b200_decompress_into(ctx, in + 4, n - 4, out, want, written, err_expected, err_actual);
}

// ---- frame format ---------------------------------------------------------------------------------

size_t lz4b200_frame_write_header(const lz4b200_frame_info *info, uint8_t *out, size_t cap)
{
    // FrameInfo::write — frame/header.rs:232-275
    uint8_t buf[19];
    size_t o = 0;
    wr32(buf, 0x184D2204u); o = 4;
    uint8_t flg = 0x40;
    if (info->block_checksums) flg |= 0x10;
    if (info->content_checksum) flg |= 0x04;
    if (!info->linked) flg |= 0x20;
    if (info->has_content_size) flg |= 0x08;
    buf[o++] = flg;
    buf[o++] = (uint8_t)(info->block_size_id << 4);
    if (info->has_content_size) { memcpy(buf + o, &info->content_size, 8); o += 8; }
    buf[o] = (uint8_t)(lz4b200_xxh32(buf + 4, o - 4, 0) >> 8);
    o++;
    if (cap < o) return 0;
    memcpy(out, buf, o);
    return o;
}

size_t lz4b200_frame_blocks_bound(size_t in_len, size_t block_size)
{
    size_t nb = block_size ? (in_len + block_size - 1) / block_size : 0;
    return in_len + nb * 4;
}

size_t lz4b200_frame_bound(size_t n, const lz4b200_frame_info *info)
{
    int id = info && info->block_size_id ? info->block_size_id : 4;
    size_t bs = block_size_bytes(id);
    if (!bs) bs = 64u << 10;
    size_t nb = (n + bs - 1) / bs;
    return 19 + n + nb * 8 + 8;
}

}  // extern "C"

namespace {

// Sets what `info` (block size resolved) and the input d_in[in_off, in_off + in_len) decide of the zeroed plan p, the
// header included; fb::plan_frame places it after the frame before.  p is filled in place, not returned: copying a
// returned plan into the batch's table stalls the host on every frame.
void frame_plan(fb::FramePlan &p, const lz4b200_frame_info &info, uint64_t in_off, uint64_t in_len)
{
    p.in_off = in_off;
    p.in_len = in_len;
    p.bs = (uint32_t)block_size_bytes(info.block_size_id);
    p.fresh = fb::fresh_period(p.bs);
    p.hdr_len = (uint8_t)lz4b200_frame_write_header(&info, p.hdr, sizeof p.hdr);
}

// The pipeline of every frame encoder: enqueues the n >= 1 frames of plan (placed by fb::plan_frame) on `s`.  One plan
// reaches the device as a kernel argument, more with one copy from pageable memory, which cudaMemcpyAsync stages before
// it returns, so back-to-back calls never share a host buffer.  Then one thread per block writes the compressor's
// arguments, one launch compresses every block of every frame, the segment sizes (with room for a checksum after each
// payload when `block_checksums`) are scanned, one gather packs every [BlockInfo | payload] at its frame's place, and
// one thread per block writes the block checksums.  max_in_len is launch_compress's bound on the blocks' lengths.  A
// device position d_pos_in moves every block *d_pos_in bytes further, and *d_pos_out receives the end of the blocks.
// With `content_checksum` one CTA per frame hashes its content; with d_frame_off one thread per frame writes its
// header, EndMark, digest (when hashed) and d_frame_off[f], and d_frame_off[n] the total.
lz4b200_status compress_frames(lz4b200_ctx *ctx, const uint8_t *d_in, const fb::FramePlan *plan, uint32_t n,
                               uint32_t max_in_len, bool block_checksums, bool content_checksum, uint8_t *d_out,
                               uint64_t *d_frame_off, const uint64_t *d_pos_in, uint64_t *d_pos_out, cudaStream_t s)
{
    const fb::FramePlan &last = plan[n - 1];
    const uint32_t nb = last.first_block + (uint32_t)fb::frame_blocks(last);
    CTX_CUDA(ctx, ctx->d_fplan.reserve(n));
    CTX_CUDA(ctx, ctx->d_slots.reserve(last.slot_base + fb::frame_slot_bytes(last) + 16));
    CTX_CUDA(ctx, ctx->d_in_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_in_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_status.reserve(nb));
    CTX_CUDA(ctx, ctx->d_flags.reserve(nb)); CTX_CUDA(ctx, ctx->d_pick.reserve(nb));
    CTX_CUDA(ctx, ctx->d_info.reserve(nb)); CTX_CUDA(ctx, ctx->d_seg_size.reserve(nb));
    CTX_CUDA(ctx, ctx->d_payload_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_seg_off.reserve((size_t)nb + 1));
    CTX_CUDA(ctx, ctx->d_gdst.reserve(nb));
    if (content_checksum) CTX_CUDA(ctx, ctx->d_content.reserve(n));
    if (n == 1) {
        frame_plan_store_kernel<<<1, 1, 0, s>>>(ctx->d_fplan.p, plan[0]);
        CTX_CUDA(ctx, cudaGetLastError());
    } else {
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_fplan.p, plan, n * sizeof(fb::FramePlan), cudaMemcpyHostToDevice, s));
    }

    const uint32_t bgrid = (nb + 127) / 128;
    if (nb) {
        frame_batch_blocks_kernel<<<bgrid, 128, 0, s>>>(ctx->d_fplan.p, n, nb, ctx->d_in_off.p, ctx->d_in_len.p,
                                                        ctx->d_out_off.p, ctx->d_out_cap.p, ctx->d_flags.p,
                                                        ctx->d_gdst.p);
        CTX_CUDA(ctx, cudaGetLastError());
        BatchArgs a{d_in, ctx->d_in_off.p, ctx->d_in_len.p, ctx->d_flags.p, ctx->d_slots.p, ctx->d_out_off.p,
                    ctx->d_out_cap.p, ctx->d_out_len.p, ctx->d_status.p, nullptr, nb, nullptr};
        const lz4b200_status st = launch_compress(ctx, a, max_in_len, s);
        if (st != LZ4B200_OK) return st;
        frame_block_info_kernel<<<(nb + 255) / 256, 256, 0, s>>>(ctx->d_out_len.p, ctx->d_in_len.p, nb,
                                                                block_checksums ? 4u : 0u, ctx->d_info.p,
                                                                ctx->d_pick.p, ctx->d_seg_size.p, ctx->d_payload_len.p);
        CTX_CUDA(ctx, cudaGetLastError());
    }
    scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_seg_size.p, ctx->d_seg_off.p, nb);   // nb == 0: seg_off[0] = 0
    CTX_CUDA(ctx, cudaGetLastError());
    if (nb) {
        frame_batch_dst_kernel<<<bgrid, 128, 0, s>>>(ctx->d_seg_off.p, nb, ctx->d_gdst.p, d_pos_in, d_pos_out);
        GatherArgs g{ctx->d_slots.p, d_in, ctx->d_out_off.p, ctx->d_in_off.p, ctx->d_payload_len.p, ctx->d_payload_len.p,
                     ctx->d_pick.p, ctx->d_info.p, d_out, ctx->d_gdst.p, nb};
        gather_segments_kernel<<<std::min<uint32_t>(std::max<uint32_t>(nb, (uint32_t)ctx->sm_count * 2),
                                                    (uint32_t)ctx->sm_count * 8), 256, 0, s>>>(g);
        CTX_CUDA(ctx, cudaGetLastError());
        if (block_checksums) {
            frame_block_checksum_kernel<<<bgrid, 128, 0, s>>>(d_out, ctx->d_gdst.p, ctx->d_payload_len.p, nb);
            CTX_CUDA(ctx, cudaGetLastError());
        }
    }
    if (content_checksum) {
        frame_batch_content_kernel<<<n, 256, 0, s>>>(d_in, ctx->d_fplan.p, ctx->d_content.p);
        CTX_CUDA(ctx, cudaGetLastError());
    }
    if (d_frame_off) {
        frame_batch_tail_kernel<<<(n + 127) / 128, 128, 0, s>>>(d_out, ctx->d_fplan.p, n, ctx->d_seg_off.p,
                                                                content_checksum ? ctx->d_content.p : nullptr,
                                                                d_frame_off);
        CTX_CUDA(ctx, cudaGetLastError());
    }
    return LZ4B200_OK;
}

}  // namespace

extern "C" {

// Rank-local half of a (possibly sharded) frame, step 1: compress the blocks of [first_block, ...) into the context's
// slots, decide compressed-vs-stored per block (frame/compress.rs:301-306) and scan the segment sizes.  *d_total
// receives the packed size.  Everything stays on the device and on `stream`.
lz4b200_status lz4b200_frame_range_compress(lz4b200_ctx *ctx, const uint8_t *d_in, size_t in_len, size_t block_size,
                                            uint64_t first_block, uint64_t *d_total, uint32_t *d_block_sizes, void *stream)
{
    if (!ctx || !block_size || block_size > (8u << 20)) return LZ4B200_INVALID_ARGUMENT;
    const size_t nblocks = (in_len + block_size - 1) / block_size;
    if (nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nb = (uint32_t)nblocks;
    ctx->range_nb = nb; ctx->range_in = d_in;
    if (nb == 0) {
        if (d_total) CTX_CUDA(ctx, cudaMemsetAsync(d_total, 0, 8, s));
        return LZ4B200_OK;
    }
    const size_t slot = (lz4b200_max_output_size(block_size) + 15) & ~size_t(15);
    CTX_CUDA(ctx, ctx->d_slots.reserve(slot * nb + 16));
    CTX_CUDA(ctx, ctx->d_in_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_in_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_status.reserve(nb));
    CTX_CUDA(ctx, ctx->d_flags.reserve(nb)); CTX_CUDA(ctx, ctx->d_pick.reserve(nb));
    CTX_CUDA(ctx, ctx->d_info.reserve(nb)); CTX_CUDA(ctx, ctx->d_seg_size.reserve(nb));
    CTX_CUDA(ctx, ctx->d_payload_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_seg_off.reserve(nb + 1));

    make_uniform_desc_kernel<<<(nb + 255) / 256, 256, 0, s>>>(in_len, (uint32_t)block_size, slot, first_block,
                                                             fb::fresh_period(block_size), nb, ctx->d_in_off.p,
                                                             ctx->d_in_len.p, ctx->d_out_off.p, ctx->d_out_cap.p,
                                                             ctx->d_flags.p);
    CTX_CUDA(ctx, cudaGetLastError());
    BatchArgs a{d_in, ctx->d_in_off.p, ctx->d_in_len.p, ctx->d_flags.p, ctx->d_slots.p, ctx->d_out_off.p,
                ctx->d_out_cap.p, ctx->d_out_len.p, ctx->d_status.p, nullptr, nb, nullptr};
    lz4b200_status st = launch_compress(ctx, a, (uint32_t)std::min<size_t>(block_size, in_len), s);
    if (st != LZ4B200_OK) return st;
    frame_block_info_kernel<<<(nb + 255) / 256, 256, 0, s>>>(ctx->d_out_len.p, ctx->d_in_len.p, nb, 0, ctx->d_info.p,
                                                            ctx->d_pick.p, ctx->d_seg_size.p, ctx->d_payload_len.p);
    CTX_CUDA(ctx, cudaGetLastError());
    scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_seg_size.p, ctx->d_seg_off.p, nb);
    CTX_CUDA(ctx, cudaGetLastError());
    if (d_total) CTX_CUDA(ctx, cudaMemcpyAsync(d_total, ctx->d_seg_off.p + nb, 8, cudaMemcpyDeviceToDevice, s));
    if (d_block_sizes)
        CTX_CUDA(ctx, cudaMemcpyAsync(d_block_sizes, ctx->d_seg_size.p, nb * 4, cudaMemcpyDeviceToDevice, s));
    return LZ4B200_OK;
}

// Step 2: pack the range's [BlockInfo | payload] segments back to back at d_dst + *d_dst_offset.  d_dst may be PEER
// memory (another GPU's frame buffer mapped over NVLink, lz4b200_peer_open): the pack kernel's stores are then the
// transfer — the per-rank chunk is never staged in local memory or handed to a separate collective.
lz4b200_status lz4b200_frame_range_pack(lz4b200_ctx *ctx, uint8_t *d_dst, const uint64_t *d_dst_offset, void *stream)
{
    if (!ctx || !d_dst) return LZ4B200_INVALID_ARGUMENT;
    const uint32_t nb = ctx->range_nb;
    if (nb == 0) return LZ4B200_OK;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    GatherArgs g{ctx->d_slots.p, ctx->range_in, ctx->d_out_off.p, ctx->d_in_off.p, ctx->d_payload_len.p, ctx->d_payload_len.p,
                 ctx->d_pick.p, ctx->d_info.p, d_dst, ctx->d_seg_off.p, nb, d_dst_offset};
    gather_segments_kernel<<<std::min<uint32_t>(std::max<uint32_t>(nb, (uint32_t)ctx->sm_count * 2), (uint32_t)ctx->sm_count * 8),
                             256, 0, s>>>(g);
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}

lz4b200_status lz4b200_frame_compress_blocks_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t in_len,
                                                    size_t block_size, uint64_t first_block, uint8_t *d_out,
                                                    size_t out_cap, uint64_t *d_total, uint32_t *d_block_sizes,
                                                    void *stream)
{
    if (!ctx || !block_size || block_size > (8u << 20)) return LZ4B200_INVALID_ARGUMENT;
    if (out_cap < lz4b200_frame_blocks_bound(in_len, block_size)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    lz4b200_status st = lz4b200_frame_range_compress(ctx, d_in, in_len, block_size, first_block, d_total, d_block_sizes, stream);
    if (st != LZ4B200_OK || in_len == 0) return st;
    return lz4b200_frame_range_pack(ctx, d_out, nullptr, stream);
}

// ---- peer-mapped buffers (CUDA IPC): rank 0 allocates the frame buffer, the other ranks of the node map it ----------
lz4b200_status lz4b200_peer_alloc(lz4b200_ctx *ctx, size_t bytes, void **d_ptr, uint8_t *handle64)
{
    if (!ctx || !d_ptr || !handle64 || !bytes) return LZ4B200_INVALID_ARGUMENT;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    DeviceGuard guard(ctx->device);
    DevBuf<uint8_t> buf;
    CTX_CUDA(ctx, buf.resize(bytes));
    cudaIpcMemHandle_t h;
    if (!ctx->check(cudaIpcGetMemHandle(&h, buf.p), "cudaIpcGetMemHandle")) return LZ4B200_CUDA_ERROR;
    memcpy(handle64, &h, 64);
    *d_ptr = std::exchange(buf.p, nullptr);
    return LZ4B200_OK;
}

lz4b200_status lz4b200_peer_open(lz4b200_ctx *ctx, const uint8_t *handle64, void **d_ptr)
{
    if (!ctx || !d_ptr || !handle64) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    CTX_CUDA(ctx, cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return LZ4B200_OK;
}

lz4b200_status lz4b200_peer_close(lz4b200_ctx *ctx, void *d_ptr)
{
    if (!ctx || !d_ptr) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    CTX_CUDA(ctx, cudaIpcCloseMemHandle(d_ptr));
    return LZ4B200_OK;
}

lz4b200_status lz4b200_peer_free(lz4b200_ctx *ctx, void *d_ptr)
{
    if (!ctx || !d_ptr) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    CTX_CUDA(ctx, cudaFree(d_ptr));
    return LZ4B200_OK;
}

// The blocks are compressed on the device: the input goes over, one plan runs through compress_frames, block checksums
// included, and the whole frame comes back.  The content digest is computed here over `in` and appended after the
// EndMark: the host core hashes faster than the device's single serial chain.
lz4b200_status lz4b200_frame_compress(lz4b200_ctx *ctx, const uint8_t *in, size_t n, const lz4b200_frame_info *info_in,
                                      size_t first_write_len, uint8_t *out, size_t cap, size_t *written)
{
    if (!ctx || !info_in || !out || !written || (!in && n)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    lz4b200_frame_info info = *info_in;
    if (info.linked) return LZ4B200_FRAME_LINKED_UNSUPPORTED;
    if (info.block_size_id == 0) info.block_size_id = auto_block_size_id(first_write_len);   // compress.rs:236-238
    if (info.block_size_id < 4 || info.block_size_id > 7) return LZ4B200_INVALID_ARGUMENT;
    if (info.has_content_size && info.content_size != n) return LZ4B200_FRAME_CONTENT_LENGTH; // compress.rs:212-219
    if (cap < lz4b200_frame_bound(n, &info)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = ctx->stream;

    fb::FramePlan plan{};
    frame_plan(plan, info, 0, n);
    CTX_CUDA(ctx, ctx->d_in.reserve(n + 16));
    CTX_CUDA(ctx, ctx->d_out.reserve(lz4b200_frame_bound(n, &info)));
    CTX_CUDA(ctx, ctx->d_off_b.reserve(2));
    if (n) CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in.p, in, n, cudaMemcpyHostToDevice, s));
    const lz4b200_status st = compress_frames(ctx, ctx->d_in.p, &plan, 1, (uint32_t)std::min<uint64_t>(n, plan.bs),
                                              info.block_checksums, false, ctx->d_out.p, ctx->d_off_b.p, nullptr, nullptr, s);
    if (st != LZ4B200_OK) return st;
    uint64_t o = 0;
    CTX_CUDA(ctx, cudaMemcpyAsync(&o, ctx->d_off_b.p + 1, 8, cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaStreamSynchronize(s));
    CTX_CUDA(ctx, cudaMemcpyAsync(out, ctx->d_out.p, o, cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaStreamSynchronize(s));
    if (info.content_checksum) { wr32(out + o, lz4b200_xxh32(in, n, 0)); o += 4; }       // compress.rs:224-227
    *written = o;
    return LZ4B200_OK;
}

// lz4b200_frame_compress for input in device memory, written to device memory without a host synchronisation: one plan
// runs through compress_frames, and the frame's end goes to *d_written.  Only kernel arguments cross PCIe.
lz4b200_status lz4b200_frame_compress_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n,
                                             const lz4b200_frame_info *info_in, size_t first_write_len, uint8_t *d_out,
                                             size_t cap, uint64_t *d_written, void *stream)
{
    if (!ctx || !info_in || !d_out || !d_written || (!d_in && n)) return LZ4B200_INVALID_ARGUMENT;
    lz4b200_frame_info info = *info_in;
    if (info.linked) return LZ4B200_FRAME_LINKED_UNSUPPORTED;
    if (info.block_size_id == 0) info.block_size_id = auto_block_size_id(first_write_len);   // compress.rs:236-238
    if (info.block_size_id < 4 || info.block_size_id > 7) return LZ4B200_INVALID_ARGUMENT;
    if (info.has_content_size && info.content_size != n) return LZ4B200_FRAME_CONTENT_LENGTH; // compress.rs:212-219
    if (cap < lz4b200_frame_bound(n, &info)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;

    fb::FramePlan plan{};
    frame_plan(plan, info, 0, n);
    CTX_CUDA(ctx, ctx->d_off_b.reserve(2));
    const lz4b200_status st = compress_frames(ctx, d_in, &plan, 1, (uint32_t)std::min<uint64_t>(n, plan.bs),
                                              info.block_checksums, info.content_checksum, d_out, ctx->d_off_b.p,
                                              nullptr, nullptr, s);
    if (st != LZ4B200_OK) return st;
    CTX_CUDA(ctx, cudaMemcpyAsync(d_written, ctx->d_off_b.p + 1, 8, cudaMemcpyDeviceToDevice, s));
    return LZ4B200_OK;
}

// lz4b200_frame_compress_device for each of many inputs, frames packed back to back, in one call: the host plans every
// frame (fb::plan_frame) and compress_frames enqueues them all on `stream`.
lz4b200_status lz4b200_frame_compress_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *in_off,
                                                   const uint64_t *in_len, const lz4b200_frame_info *info,
                                                   uint8_t *d_out, size_t out_cap, uint64_t *d_frame_off,
                                                   size_t nframes, void *stream)
{
    if (!ctx || !info || !d_frame_off || (nframes && (!in_off || !in_len || !d_out))) return LZ4B200_INVALID_ARGUMENT;
    if (!d_in)
        for (size_t f = 0; f < nframes; f++)
            if (in_len[f]) return LZ4B200_INVALID_ARGUMENT;
    if (info->linked) return LZ4B200_FRAME_LINKED_UNSUPPORTED;
    const int id = info->block_size_id;
    if ((id != 0 && (id < 4 || id > 7)) || nframes > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    const uint32_t tail = info->content_checksum ? 8u : 4u;
    std::vector<fb::FramePlan> plan(nframes);
    uint64_t nblocks = 0, bound = 0, max_len = 0;
    bool small = false;                                     // some block has at most 64 KiB
    for (size_t f = 0; f < nframes; f++) {
        lz4b200_frame_info fi = *info;
        if (id == 0) fi.block_size_id = auto_block_size_id(in_len[f]);                      // compress.rs:236-238
        fi.content_size = in_len[f];
        fb::FramePlan &p = plan[f];
        frame_plan(p, fi, in_off[f], in_len[f]);
        const uint64_t nb = fb::frame_blocks(p);
        if (nblocks + nb > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
        fb::plan_frame(p, f ? &plan[f - 1] : nullptr, tail);
        nblocks += nb;
        bound += lz4b200_frame_bound(p.in_len, &fi);
        if (nb) {
            max_len = std::max<uint64_t>(max_len, std::min<uint64_t>(p.in_len, p.bs));
            small = small || p.in_len - (nb - 1) * p.bs <= 65536u;               // the last block is the shortest
        }
    }
    if (out_cap < bound) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    if (nframes == 0) {
        CTX_CUDA(ctx, cudaMemsetAsync(d_frame_off, 0, 8, s));
        return LZ4B200_OK;
    }
    // blocks on both sides of 64 KiB run both encoders whatever the bound says; an unknown bound (0) makes the
    // launcher's record name both
    const uint32_t max_in_len = small && max_len > 65536u ? 0u : (uint32_t)max_len;
    return compress_frames(ctx, d_in, plan.data(), (uint32_t)nframes, max_in_len, info->block_checksums,
                           info->content_checksum, d_out, d_frame_off, nullptr, nullptr, s);
}

namespace {

constexpr uint32_t kHostWalkChunk = 4096;     // descriptors per frame_walk() call on the host
constexpr uint32_t kDeviceWalkChunk = 65536;  // descriptors one walk launch records on the device (16 B each)

// The frame at in[0, n) in host memory: header and BlockInfo chain.
void walk_frame_host(const uint8_t *in, size_t n, fw::FrameWalk &w, std::vector<fw::FrameBlockDesc> &blocks)
{
    w = fw::FrameWalk{};
    blocks.clear();
    while (w.stage != fw::kWalkDone) {
        const size_t at = blocks.size();
        blocks.resize(at + kHostWalkChunk);
        blocks.resize(at + fw::frame_walk(in, n, w, blocks.data() + at, kHostWalkChunk));
    }
}

// The block checksum step on the host: the first recorded block whose stored checksum is wrong, or kNoBlock.
uint32_t first_bad_block_host(const uint8_t *in, const fw::FrameWalk &w, const std::vector<fw::FrameBlockDesc> &blocks)
{
    if (!(w.flg & 0x10)) return fw::kNoBlock;
    for (size_t k = 0; k < blocks.size(); k++)
        if (!fw::block_checksum_ok(in, blocks[k])) return (uint32_t)k;
    return fw::kNoBlock;
}

// The frame at d_in[0, n) in device memory: the walk runs in one GPU thread, kDeviceWalkChunk blocks per launch; only
// the walk state and the descriptors (16 B per block) come back to the host.  With `verify`, each launch's blocks have
// their checksums checked on the device and *bad receives the first failing block (kNoBlock: none).
lz4b200_status walk_frame_device(lz4b200_ctx *ctx, cudaStream_t s, const uint8_t *d_in, size_t n, bool verify,
                                 fw::FrameWalk &w, std::vector<fw::FrameBlockDesc> &blocks, uint32_t *bad)
{
    w = fw::FrameWalk{};
    blocks.clear();
    *bad = fw::kNoBlock;
    CTX_CUDA(ctx, ctx->d_walk.reserve(1)); CTX_CUDA(ctx, ctx->d_desc.reserve(kDeviceWalkChunk));
    CTX_CUDA(ctx, ctx->d_bad.reserve(1));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_walk.p, &w, sizeof w, cudaMemcpyHostToDevice, s));
    if (verify) CTX_CUDA(ctx, cudaMemsetAsync(ctx->d_bad.p, 0xff, 4, s));
    while (w.stage != fw::kWalkDone) {
        const uint64_t first = w.nblocks;
        frame_walk_kernel<<<1, 1, 0, s>>>(d_in, n, ctx->d_walk.p, ctx->d_desc.p, kDeviceWalkChunk);
        CTX_CUDA(ctx, cudaGetLastError());
        if (verify) {
            block_checksum_kernel<<<kDeviceWalkChunk / 128, 128, 0, s>>>(d_in, ctx->d_desc.p, ctx->d_walk.p, first, ctx->d_bad.p);
            CTX_CUDA(ctx, cudaGetLastError());
        }
        CTX_CUDA(ctx, cudaMemcpyAsync(&w, ctx->d_walk.p, sizeof w, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
        const size_t k = w.nblocks - first;
        blocks.resize(first + k);
        if (k) {
            CTX_CUDA(ctx, cudaMemcpyAsync(blocks.data() + first, ctx->d_desc.p, k * sizeof(fw::FrameBlockDesc),
                                          cudaMemcpyDeviceToHost, s));
            CTX_CUDA(ctx, cudaStreamSynchronize(s));
        }
    }
    if (verify && !blocks.empty()) {
        CTX_CUDA(ctx, cudaMemcpyAsync(bad, ctx->d_bad.p, 4, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
    }
    return LZ4B200_OK;
}

// Every concatenated frame of in[0, n) (host or, with `device`, device memory), summed over the blocks each walk records.
// The header's content_size is NOT used: it is untrusted, and a frame whose real size differs must still be delivered
// in full before ContentLengthError is reported (frame/decompress.rs:312-321).
lz4b200_status frame_decoded_bound_impl(lz4b200_ctx *ctx, cudaStream_t s, bool device, const uint8_t *in, size_t n,
                                        size_t *bound)
{
    fw::FrameWalk w;
    std::vector<fw::FrameBlockDesc> blocks;
    size_t ip = 0, total = 0;
    while (ip < n) {
        if (device) {
            uint32_t bad;
            const lz4b200_status st = walk_frame_device(ctx, s, in + ip, n - ip, false, w, blocks, &bad);
            if (st != LZ4B200_OK) return st;
        } else {
            walk_frame_host(in + ip, n - ip, w, blocks);
        }
        for (const fw::FrameBlockDesc &b : blocks)
            total += fw::block_stored(b) ? fw::block_len(b) : (size_t)fw::block_decoded_cap(fw::block_len(b), w.bs);
        if (w.status != LZ4B200_OK || !w.closed) break;
        ip += w.ip;
    }
    *bound = total;
    return LZ4B200_OK;
}

// The group pipeline (see GroupFrame) over the gn frames at ctx->d_gframe, whose nb blocks (the nind independent ones
// first) are described at ctx->d_desc and ctx->d_bframe and whose slots take `slots` bytes: payload read at src, output
// gathered into out.  Everything is enqueued on s.
lz4b200_status decode_group(lz4b200_ctx *ctx, cudaStream_t s, const uint8_t *src, uint8_t *out, uint32_t gn, uint32_t nb,
                            uint32_t nind, uint64_t slots)
{
    const uint32_t nlnk = nb - nind, fgrid = (gn + 127) / 128, bgrid = (nb + 127) / 128;
    GroupFrame *frames = ctx->d_gframe.p;
    CTX_CUDA(ctx, ctx->d_fhash.reserve(gn));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb + 1)); CTX_CUDA(ctx, ctx->d_slots.reserve(slots + 16));
    CTX_CUDA(ctx, ctx->d_in_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_in_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_status.reserve(nb)); CTX_CUDA(ctx, ctx->d_expected.reserve(nb));
    CTX_CUDA(ctx, ctx->d_pick.reserve(nb)); CTX_CUDA(ctx, ctx->d_link_first.reserve(nb));
    CTX_CUDA(ctx, ctx->d_stored_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_done.reserve(nb));
    CTX_CUDA(ctx, ctx->d_bslot.reserve(nb)); CTX_CUDA(ctx, ctx->d_gdst.reserve(nb)); CTX_CUDA(ctx, ctx->d_glen.reserve(nb));
    if (nb) {
        frame_batch_args_kernel<<<bgrid, 128, 0, s>>>(frames, ctx->d_desc.p, ctx->d_bframe.p, nb, nind, ctx->d_in_off.p,
                                                      ctx->d_in_len.p, ctx->d_out_cap.p, ctx->d_pick.p,
                                                      ctx->d_link_first.p, ctx->d_stored_len.p, ctx->d_done.p,
                                                      ctx->d_bslot.p);
        scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_bslot.p, ctx->d_out_off.p, nb);
        CTX_CUDA(ctx, cudaGetLastError());
        BatchArgs a{src, ctx->d_in_off.p, ctx->d_in_len.p, nullptr, ctx->d_slots.p, ctx->d_out_off.p,
                    ctx->d_out_cap.p, ctx->d_out_len.p, ctx->d_status.p, ctx->d_expected.p, nind, nullptr};
        const lz4b200_status st = launch_decompress(ctx, a, s);
        if (st != LZ4B200_OK) return st;
        if (nlnk) {
            // BlockMode::Linked (frame/decompress.rs:196-222): every linked chain of the group in one launch; block b
            // waits only for blocks [link_first[b], b) of its frame and resolves offsets that reach before it in their
            // outputs
            BatchArgs l{src, ctx->d_in_off.p + nind, ctx->d_in_len.p + nind, nullptr, ctx->d_slots.p,
                        ctx->d_out_off.p + nind, ctx->d_out_cap.p + nind, ctx->d_out_len.p + nind,
                        ctx->d_status.p + nind, ctx->d_expected.p + nind, nlnk, ctx->d_tickets.p};
            l.link_first = ctx->d_link_first.p + nind; l.stored_off = ctx->d_in_off.p + nind;
            l.stored_len = ctx->d_stored_len.p + nind; l.done = ctx->d_done.p + nind;
            lz4_decompress_blocks_linked<32><<<std::min<uint32_t>((nlnk + 3) / 4, (uint32_t)ctx->sm_count * 8), 128, 0, s>>>(l);
            CTX_CUDA(ctx, cudaGetLastError());
        }
    }
    frame_resolve_kernel<<<(gn + 3) / 4, 128, 0, s>>>(frames, gn, ctx->d_desc.p, ctx->d_out_len.p, ctx->d_status.p,
                                               ctx->d_expected.p, ctx->d_out_cap.p, ctx->d_gdst.p, ctx->d_glen.p,
                                               ctx->d_fhash.p);
    CTX_CUDA(ctx, cudaGetLastError());
    if (nb) {
        GatherArgs g{ctx->d_slots.p, src, ctx->d_out_off.p, ctx->d_in_off.p, ctx->d_glen.p, ctx->d_glen.p,
                     ctx->d_pick.p, nullptr, out, ctx->d_gdst.p, nb};
        gather_segments_kernel<<<std::min<uint32_t>(nb, (uint32_t)ctx->sm_count * 8), 256, 0, s>>>(g);
        CTX_CUDA(ctx, cudaGetLastError());
    }
    frame_batch_hash_kernel<<<gn, 256, 0, s>>>(out, frames, ctx->d_fhash.p);
    frame_batch_digest_kernel<<<fgrid, 128, 0, s>>>(frames, gn, ctx->d_fhash.p);
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}

// Decodes the blocks a walk `w` recorded through the group pipeline, in groups whose device slots fit the context's
// frame budget (slots are reused from group to group), so a frame of many short blocks costs O(budget) device memory,
// not #blocks x block size.  `in` and `out` are host memory (each group's payload is staged to the device and its
// output copied back), or with `device` device memory, read and written in place.  The frame delivered `delivered`
// bytes before blocks[0], whose output goes to out[0]; `last`: the blocks end the frame.  `content` carries the
// frame's content hash: device memory, or with host memory (`device` false) the host hashes each group's output as it
// lands and the caller compares the digest (one CPU core hashes faster than the GPU's one XXH32 chain).  *r receives the frame's result after the last group decoded (the first that does
// not return LZ4B200_OK stops the loop), and so does *d_result (device memory) if not null.
// A linked frame's blocks may continue one decoded earlier (the streaming decoder, device memory only): `window` holds
// the last `window_len` (<= 64 KiB) bytes of the frame's output before blocks[0], and the linked kernel sees it as a
// stored block ahead of the group, staged with the group's payload in one buffer.  On FRAME_DECOMPRESSION_ERROR,
// *failed (if not null) receives the index of the block that failed.
lz4b200_status decode_frame_blocks(lz4b200_ctx *ctx, cudaStream_t s, bool device, const uint8_t *in, uint8_t *out,
                                   size_t cap, const fw::FrameWalk &w, const std::vector<fw::FrameBlockDesc> &blocks,
                                   bool last, uint64_t delivered, lz4b200_xxh32_state *content, lz4b200_frame_result *r,
                                   lz4b200_frame_result *d_result = nullptr, const uint8_t *window = nullptr,
                                   uint32_t window_len = 0, uint32_t *failed = nullptr)
{
    const uint32_t nb = (uint32_t)blocks.size();
    *r = lz4b200_frame_result{};
    r->written = delivered;
    if (!nb && !last) return LZ4B200_OK;                                 // nothing to decode and nothing to decide
    DeviceGuard guard(ctx->device);
    const bool linked = nb && w.linked && (nb > 1 || window_len > 0);
    const uint32_t pre = linked && window_len ? 1 : 0;                   // the window's pseudo-block ahead of the group
    CTX_CUDA(ctx, ctx->d_walk.reserve(1)); CTX_CUDA(ctx, ctx->d_gframe.reserve(1)); CTX_CUDA(ctx, ctx->d_result.reserve(1));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_walk.p, &w, sizeof w, cudaMemcpyHostToDevice, s));
    uint64_t got = 0;                                                     // the bytes delivered from blocks[0] on
    uint32_t g0 = 0;
    do {
        // a group: as many blocks as fit the budget (a linked frame is one dependency chain: one group)
        uint32_t g1 = g0;
        uint64_t slot_total = 0;
        while (g1 < nb) {
            const uint64_t c = fw::block_slot_cap(blocks[g1], w.bs);
            const uint64_t in_span = blocks[g1].payload_off + fw::block_len(blocks[g1]) - blocks[g0].payload_off;
            if (!linked && g1 > g0 && fw::group_cut(slot_total, c, in_span, ctx->frame_budget)) break;
            slot_total += fw::slot_bytes(c);
            g1++;
        }
        const uint32_t gn = g1 - g0, gm = gn + pre;                      // the kernel's blocks: [window,] the group
        const uint64_t in_lo = gn ? blocks[g0].payload_off : 0;
        const uint64_t in_bytes = gn ? blocks[g1 - 1].payload_off + fw::block_len(blocks[g1 - 1]) - in_lo : 0;
        const uint64_t shift = pre ? window_len : 0;                       // the payload's place in a staged buffer
        GroupFrame p{};
        const uint8_t *src = in;                                           // the frame's payload on the device
        if (gn && (!device || pre)) {
            CTX_CUDA(ctx, ctx->d_in.reserve(shift + in_bytes + 16));
            if (pre) CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in.p, window, window_len, cudaMemcpyDeviceToDevice, s));
            CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in.p + shift, in + in_lo, in_bytes,
                                          device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s));
            src = ctx->d_in.p;
            p.in_off = shift - in_lo;                                      // mod 2^64: payload offsets add back to it
        }
        uint8_t *dst = out;                                                // the device path gathers in place
        if (device) {
            p.out_off = got;
        } else {
            CTX_CUDA(ctx, ctx->d_out.reserve(std::min<uint64_t>(cap - got, slot_total + in_bytes) + 16));
            dst = ctx->d_out.p;
        }
        p.out_cap = cap - got;
        p.delivered = delivered + got;
        p.walk = ctx->d_walk.p;
        p.content = device ? content : nullptr;
        p.result = d_result ? d_result : ctx->d_result.p;
        p.nblocks = gm;
        p.bad = fw::kNoBlock;
        p.window = (uint8_t)pre;
        p.last = last && g1 == nb;
        CTX_CUDA(ctx, ctx->d_desc.reserve(gm)); CTX_CUDA(ctx, ctx->d_bframe.reserve(gm));
        if (pre) {
            const fw::FrameBlockDesc wd{in_lo - shift, window_len | 0x80000000u, 0};   // stored at the staged buffer's start
            CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_desc.p, &wd, sizeof wd, cudaMemcpyHostToDevice, s));
        }
        if (gn) CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_desc.p + pre, blocks.data() + g0, gn * sizeof(fw::FrameBlockDesc),
                                              cudaMemcpyHostToDevice, s));
        CTX_CUDA(ctx, cudaMemsetAsync(ctx->d_bframe.p, 0, gm * sizeof(uint32_t), s));
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_gframe.p, &p, sizeof p, cudaMemcpyHostToDevice, s));
        const lz4b200_status st = decode_group(ctx, s, src, dst, 1, gm, linked ? 0 : gm, slot_total);
        if (st != LZ4B200_OK) return st;
        uint32_t bad = fw::kNoBlock;
        CTX_CUDA(ctx, cudaMemcpyAsync(r, p.result, sizeof *r, cudaMemcpyDeviceToHost, s));
        if (failed) CTX_CUDA(ctx, cudaMemcpyAsync(&bad, &ctx->d_gframe.p->bad, sizeof bad, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
        const uint64_t n = r->written - p.delivered;
        if (!device && n) {
            CTX_CUDA(ctx, cudaMemcpyAsync(out + got, ctx->d_out.p, n, cudaMemcpyDeviceToHost, s));
            CTX_CUDA(ctx, cudaStreamSynchronize(s));
            if (w.flg & 0x04) fw::xxh32_update(*content, out + got, n);
        }
        got += n;
        if (failed && r->status == LZ4B200_FRAME_DECOMPRESSION_ERROR) *failed = g0 + bad;
        g0 = g1;
    } while (r->status == LZ4B200_OK && g0 < nb);
    return LZ4B200_OK;
}

// One frame, FrameDecoder::read_to_end (frame/decompress.rs:109-342): walk, block checksums, then the group loop, whose
// last group decides the content size and checksum at the EndMark.  `in` and `out` are host memory, or device memory
// with `device`; both paths run the same walk and the same group loop, so they return the same result for the same
// bytes.  *d_result (device memory), if not null, also receives the result.
lz4b200_status frame_decompress_next_impl(lz4b200_ctx *ctx, cudaStream_t s, bool device, const uint8_t *in, size_t n,
                                          uint8_t *out, size_t cap, size_t *consumed, size_t *written, int *block_status,
                                          uint64_t *err_expected, uint64_t *err_actual,
                                          lz4b200_frame_result *d_result = nullptr)
{
    *written = 0; *consumed = 0;
    if (block_status) *block_status = 0;
    if (err_expected) *err_expected = 0;
    if (err_actual) *err_actual = 0;
    if (n == 0) return LZ4B200_OK;                          // read_frame_info: 0 bytes where a frame would start = end of data

    fw::FrameWalk w;
    std::vector<fw::FrameBlockDesc> blocks;
    uint32_t bad = fw::kNoBlock;
    if (device) {
        const lz4b200_status st = walk_frame_device(ctx, s, in, n, true, w, blocks, &bad);
        if (st != LZ4B200_OK) return st;
    } else {
        walk_frame_host(in, n, w, blocks);
        bad = first_bad_block_host(in, w, blocks);
    }
    if (bad != fw::kNoBlock) {                               // the frame ends at the first block that fails its checksum
        fw::frame_walk_fail_block(w, blocks[bad], bad);
        blocks.resize(bad);
    }
    *consumed = w.ip;
    lz4b200_xxh32_state host_content;
    fw::xxh32_reset(host_content, 0);
    if (device) CTX_CUDA(ctx, ctx->d_content.reserve(1));
    lz4b200_frame_result r;
    const lz4b200_status st = decode_frame_blocks(ctx, s, device, in, out, cap, w, blocks, true, 0,
                                                  device ? ctx->d_content.p : &host_content, &r, d_result);
    *written = r.written;
    if (st != LZ4B200_OK) return st;
    if (!device && r.status == LZ4B200_OK && w.closed && w.has_checksum &&
        fw::xxh32_digest(host_content) != w.content_checksum)
        r.status = LZ4B200_FRAME_CONTENT_CHECKSUM;           // the digest kernel's rule, for the host's hash
    if (block_status) *block_status = r.block_status;
    if (err_expected) *err_expected = r.err_expected;
    if (err_actual) *err_actual = r.err_actual;
    return (lz4b200_status)r.status;
}

// A group of the batch: frames [f0, f0 + gn), each of which the group loop decodes as one group, with nind blocks of
// independent frames and nlnk of linked frames whose slots take `slots` bytes.  Record walk and block checksums, then
// the group pipeline, all enqueued on s.
lz4b200_status decode_frame_group(lz4b200_ctx *ctx, cudaStream_t s, const uint8_t *d_in, const uint64_t *d_frame_off,
                                  const uint64_t *d_frame_len, uint8_t *d_out, const uint64_t *d_out_off,
                                  const uint64_t *d_out_cap, lz4b200_frame_result *d_results, uint32_t nframes,
                                  uint32_t f0, uint32_t gn, uint32_t nind, uint32_t nlnk, uint64_t slots)
{
    const uint32_t nb = nind + nlnk;
    CTX_CUDA(ctx, ctx->d_fscan.reserve(2 * (size_t)(gn + 1))); CTX_CUDA(ctx, ctx->d_gframe.reserve(gn));
    CTX_CUDA(ctx, ctx->d_content.reserve(gn));
    CTX_CUDA(ctx, ctx->d_desc.reserve(nb)); CTX_CUDA(ctx, ctx->d_bframe.reserve(nb));
    uint64_t *scan_ind = ctx->d_fscan.p, *scan_lnk = ctx->d_fscan.p + gn + 1;

    scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_fnb.p + f0, scan_ind, gn);
    scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_fnb.p + nframes + f0, scan_lnk, gn);
    frame_record_kernel<<<(gn + 127) / 128, 128, 0, s>>>(d_in, d_frame_off, d_frame_len, d_out_off, d_out_cap, f0, gn,
                                                         ctx->d_fwalk.p, ctx->d_fcount.p, scan_ind, scan_lnk,
                                                         ctx->d_desc.p, ctx->d_bframe.p, ctx->d_content.p, d_results,
                                                         ctx->d_gframe.p);
    if (nb) frame_batch_checksum_kernel<<<(nb + 127) / 128, 128, 0, s>>>(d_in, ctx->d_desc.p, ctx->d_bframe.p, nb,
                                                                        ctx->d_gframe.p);
    CTX_CUDA(ctx, cudaGetLastError());
    return decode_group(ctx, s, d_in, d_out, gn, nb, nind, slots);
}

}  // namespace

lz4b200_status lz4b200_frame_decoded_bound(const uint8_t *in, size_t n, size_t *bound)
{
    if (!bound || (!in && n)) return LZ4B200_INVALID_ARGUMENT;
    return frame_decoded_bound_impl(nullptr, nullptr, false, in, n, bound);
}

lz4b200_status lz4b200_frame_decoded_bound_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n, size_t *bound,
                                                  void *stream)
{
    if (!ctx || !bound || (!d_in && n)) return LZ4B200_INVALID_ARGUMENT;
    *bound = 0;
    DeviceGuard guard(ctx->device);
    return frame_decoded_bound_impl(ctx, (cudaStream_t)stream, true, d_in, n, bound);
}

void lz4b200_ctx_set_frame_budget(lz4b200_ctx *ctx, size_t bytes)
{
    if (ctx) ctx->frame_budget = std::max<size_t>(bytes, 1u << 20);
}

// One frame from host memory into host memory: the walk and the block / content checksums on the CPU, each group's
// payload staged to the device, decoded, and copied back.
lz4b200_status lz4b200_frame_decompress_next(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                             size_t *consumed, size_t *written, int *block_status,
                                             uint64_t *err_expected, uint64_t *err_actual)
{
    if (!ctx || !written || !consumed || (!in && n) || (!out && cap)) return LZ4B200_INVALID_ARGUMENT;
    return frame_decompress_next_impl(ctx, ctx->stream, false, in, n, out, cap, consumed, written, block_status,
                                      err_expected, err_actual);
}

// One frame from device memory into device memory: walk, block checksums, decode and content checksum on the GPU; only
// the walk, block descriptors and one result per group cross PCIe.
lz4b200_status lz4b200_frame_decompress_next_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n, uint8_t *d_out,
                                                    size_t cap, size_t *consumed, size_t *written, int *block_status,
                                                    uint64_t *err_expected, uint64_t *err_actual, void *stream)
{
    if (!ctx || !written || !consumed || (!d_in && n) || (!d_out && cap)) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    const lz4b200_status st = frame_decompress_next_impl(ctx, s, true, d_in, n, d_out, cap, consumed, written,
                                                         block_status, err_expected, err_actual);
    if (st != LZ4B200_CUDA_ERROR) CTX_CUDA(ctx, cudaStreamSynchronize(s));
    return st;
}

// Many frames from device memory into device memory.  One thread per frame counts its blocks; the host cuts the batch
// into groups of whole frames whose slots fit the frame budget, each decoded as the one-frame group loop would decode
// the frame, but with every frame's blocks in the same launches.  A frame that the group loop would split into several
// groups (at least one budget of slots) goes through the one-frame device call instead.
lz4b200_status lz4b200_frame_decompress_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_frame_off,
                                                     const uint64_t *d_frame_len, uint8_t *d_out,
                                                     const uint64_t *d_out_off, const uint64_t *d_out_cap,
                                                     lz4b200_frame_result *d_results, size_t nframes, void *stream)
{
    if (!ctx || nframes > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nframes && (!d_in || !d_frame_off || !d_frame_len || !d_out || !d_out_off || !d_out_cap || !d_results))
        return LZ4B200_INVALID_ARGUMENT;
    if (!nframes) return LZ4B200_OK;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t n = (uint32_t)nframes;
    CTX_CUDA(ctx, ctx->d_fwalk.reserve(n)); CTX_CUDA(ctx, ctx->d_fcount.reserve(n));
    CTX_CUDA(ctx, ctx->d_fnb.reserve(2 * (size_t)n));
    frame_count_kernel<<<(n + 127) / 128, 128, 0, s>>>(d_in, d_frame_off, d_frame_len, n, ctx->frame_budget,
                                                       ctx->d_fwalk.p, ctx->d_fcount.p, ctx->d_fnb.p);
    CTX_CUDA(ctx, cudaGetLastError());
    std::vector<fw::FrameCount> counts(n);
    CTX_CUDA(ctx, cudaMemcpyAsync(counts.data(), ctx->d_fcount.p, n * sizeof(fw::FrameCount), cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaStreamSynchronize(s));

    // groups of consecutive one-group frames whose slots fit the budget (a linked frame larger than the budget is a group
    // of its own, as in the group loop); at most kGroupItems frames plus blocks per group bound the descriptor arrays
    constexpr uint64_t kGroupItems = 1u << 20;
    std::vector<uint32_t> solo;
    uint32_t g0 = 0, nind = 0, nlnk = 0;                   // the open group is frames [g0, f)
    uint64_t slots = 0, items = 0;
    auto flush = [&](uint32_t f) {
        const lz4b200_status st = f > g0 ? decode_frame_group(ctx, s, d_in, d_frame_off, d_frame_len, d_out, d_out_off,
                                                              d_out_cap, d_results, n, g0, f - g0, nind, nlnk, slots)
                                         : LZ4B200_OK;
        g0 = f; nind = nlnk = 0; slots = items = 0;
        return st;
    };
    for (uint32_t f = 0; f < n; f++) {
        const fw::FrameCount &c = counts[f];
        const bool batch = c.one_group && c.nblocks < kGroupItems;
        if (!batch || slots + c.slot_total > ctx->frame_budget || items + 1 + c.nblocks > kGroupItems) {
            const lz4b200_status st = flush(f);
            if (st != LZ4B200_OK) return st;
        }
        if (!batch) { solo.push_back(f); g0 = f + 1; continue; }
        (c.linked ? nlnk : nind) += (uint32_t)c.nblocks;
        slots += c.slot_total;
        items += 1 + c.nblocks;
    }
    const lz4b200_status st = flush(n);
    if (st != LZ4B200_OK) return st;
    if (!solo.empty()) {
        // frames the group loop splits (at least one budget of slots) or with more blocks than a group holds: the
        // one-frame device call, which runs the group loop over them and writes their results on the device (every such
        // frame has blocks, so the loop runs)
        std::vector<uint64_t> off(n), len(n), ooff(n), ocap(n);
        CTX_CUDA(ctx, cudaMemcpyAsync(off.data(), d_frame_off, n * 8ull, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaMemcpyAsync(len.data(), d_frame_len, n * 8ull, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaMemcpyAsync(ooff.data(), d_out_off, n * 8ull, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaMemcpyAsync(ocap.data(), d_out_cap, n * 8ull, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
        for (const uint32_t f : solo) {
            size_t consumed = 0, written = 0;
            if (frame_decompress_next_impl(ctx, s, true, d_in + off[f], len[f], d_out + ooff[f], ocap[f], &consumed,
                                           &written, nullptr, nullptr, nullptr, d_results + f) == LZ4B200_CUDA_ERROR)
                return LZ4B200_CUDA_ERROR;
        }
    }
    CTX_CUDA(ctx, cudaStreamSynchronize(s));
    return LZ4B200_OK;
}

// lz4b200_frame_decoded_bound of the first frame of every region, on the GPU; enqueued on `stream`.
lz4b200_status lz4b200_frame_decoded_bound_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in,
                                                        const uint64_t *d_frame_off, const uint64_t *d_frame_len,
                                                        uint64_t *d_bound, size_t nframes, void *stream)
{
    if (!ctx || nframes > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nframes && (!d_in || !d_frame_off || !d_frame_len || !d_bound)) return LZ4B200_INVALID_ARGUMENT;
    if (!nframes) return LZ4B200_OK;
    DeviceGuard guard(ctx->device);
    const uint32_t n = (uint32_t)nframes;
    frame_bound_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(d_in, d_frame_off, d_frame_len, n, d_bound);
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}

// Every concatenated frame of `in`, back to back (a convenience over lz4b200_frame_decompress_next: the reference's
// reader stops at each EndMark, frame/decompress.rs:310-331, and a caller that cares about frame boundaries uses _next).
lz4b200_status lz4b200_frame_decompress(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                        size_t *written, int *block_status)
{
    if (!ctx || !written || (!in && n) || (!out && cap)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (block_status) *block_status = 0;
    size_t ip = 0;
    while (ip < n) {
        size_t used = 0, w = 0;
        const lz4b200_status st = lz4b200_frame_decompress_next(ctx, in + ip, n - ip, out + *written, cap - *written, &used,
                                                                &w, block_status, nullptr, nullptr);
        *written += w;
        if (st != LZ4B200_OK) return st;
        if (used == 0) break;
        ip += used;
    }
    return LZ4B200_OK;
}

// ---- frame index and range decode (no lz4_flex counterpart) ------------------------------------------------------------
// The index: the one-frame device walk and block checksums, one sizing thread per block, then the frame decoders' own
// result step (frame_resolve_kernel) over the sizes, so the index decides its result by the rules the decoders use.
lz4b200_status lz4b200_frame_index_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n,
                                          lz4b200_frame_index_entry *d_index, size_t max_blocks, size_t *nblocks,
                                          lz4b200_frame_index_info *info, void *stream)
{
    if (!ctx || !nblocks || (!d_in && n) || (d_index && !info)) return LZ4B200_INVALID_ARGUMENT;
    *nblocks = 0;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    fw::FrameWalk w;
    std::vector<fw::FrameBlockDesc> blocks;
    uint32_t bad = fw::kNoBlock;
    lz4b200_status st = walk_frame_device(ctx, s, d_in, n, d_index != nullptr, w, blocks, &bad);
    if (st != LZ4B200_OK) return st;
    if (bad != fw::kNoBlock) {                               // the frame ends at the first block that fails its checksum
        fw::frame_walk_fail_block(w, blocks[bad], bad);
        blocks.resize(bad);
    }
    *nblocks = blocks.size();
    if (!d_index) return LZ4B200_OK;
    if (max_blocks < blocks.size() || blocks.size() >= 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    const uint32_t nb = (uint32_t)blocks.size(), grid = (nb + 127) / 128;
    CTX_CUDA(ctx, ctx->d_walk.reserve(1)); CTX_CUDA(ctx, ctx->d_gframe.reserve(1)); CTX_CUDA(ctx, ctx->d_result.reserve(1));
    CTX_CUDA(ctx, ctx->d_fhash.reserve(1)); CTX_CUDA(ctx, ctx->d_desc.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_status.reserve(nb)); CTX_CUDA(ctx, ctx->d_expected.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb)); CTX_CUDA(ctx, ctx->d_reach.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb + 1)); CTX_CUDA(ctx, ctx->d_gdst.reserve(nb)); CTX_CUDA(ctx, ctx->d_glen.reserve(nb));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_walk.p, &w, sizeof w, cudaMemcpyHostToDevice, s));
    if (nb) {
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_desc.p, blocks.data(), nb * sizeof(fw::FrameBlockDesc), cudaMemcpyHostToDevice, s));
        fr::block_size_kernel<<<grid, 128, 0, s>>>(d_in, ctx->d_desc.p, nb, w.bs, w.linked != 0, ctx->d_out_len.p,
                                                   ctx->d_status.p, ctx->d_expected.p, ctx->d_out_cap.p, ctx->d_reach.p);
        if (w.linked) {
            scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_out_len.p, ctx->d_out_off.p, nb);
            fr::block_reach_kernel<<<grid, 128, 0, s>>>(ctx->d_out_off.p, ctx->d_reach.p, nb, ctx->d_status.p,
                                                        ctx->d_expected.p, ctx->d_out_len.p);
        }
        CTX_CUDA(ctx, cudaGetLastError());
    }
    GroupFrame p{};
    p.out_cap = ~0ull;                                        // a sufficient cap
    p.walk = ctx->d_walk.p;
    p.result = ctx->d_result.p;
    p.nblocks = nb;
    p.bad = fw::kNoBlock;
    p.last = 1;
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_gframe.p, &p, sizeof p, cudaMemcpyHostToDevice, s));
    frame_resolve_kernel<<<1, 128, 0, s>>>(ctx->d_gframe.p, 1, ctx->d_desc.p, ctx->d_out_len.p, ctx->d_status.p,
                                           ctx->d_expected.p, ctx->d_out_cap.p, ctx->d_gdst.p, ctx->d_glen.p, ctx->d_fhash.p);
    if (nb) fr::index_entries_kernel<<<grid, 128, 0, s>>>(ctx->d_desc.p, ctx->d_gdst.p, ctx->d_glen.p, nb, d_index);
    CTX_CUDA(ctx, cudaGetLastError());
    lz4b200_frame_result r;
    uint32_t failed = fw::kNoBlock;
    CTX_CUDA(ctx, cudaMemcpyAsync(&r, ctx->d_result.p, sizeof r, cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaMemcpyAsync(&failed, &ctx->d_gframe.p->bad, sizeof failed, cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaStreamSynchronize(s));
    *info = lz4b200_frame_index_info{};
    info->block_size = w.bs;
    info->nblocks = std::min(nb, failed);
    info->content_len = r.written;
    info->linked = w.linked;
    info->result = r;
    return LZ4B200_OK;
}

namespace {

constexpr uint32_t kRangeChunk = 65536;                      // ranges planned per launch
constexpr uint32_t kRangeItems = 65536;                      // (range, block) items per decode launch, at most

// Independent blocks: per chunk of ranges, a plan (first block, block count, item offsets) and one readback of the item
// count; then windows of items whose partial-block slots fit the frame budget, each decoded, checked and copied.
lz4b200_status decode_ranges_independent(lz4b200_ctx *ctx, cudaStream_t s, const uint8_t *d_in,
                                         const lz4b200_frame_index_info &info, const lz4b200_frame_index_entry *d_index,
                                         const uint64_t *d_start, const uint64_t *d_len, uint8_t *d_out,
                                         const uint64_t *d_out_off, uint64_t *d_written, uint32_t nr)
{
    const uint32_t nb = (uint32_t)info.nblocks;
    const uint64_t slot = fw::slot_bytes(info.block_size);
    const uint32_t K = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>(kRangeItems, ctx->frame_budget / std::max<uint64_t>(slot, 1)));
    CTX_CUDA(ctx, ctx->d_rfirst.reserve(kRangeChunk)); CTX_CUDA(ctx, ctx->d_rcount.reserve(kRangeChunk));
    CTX_CUDA(ctx, ctx->d_ritem.reserve(kRangeChunk + 1));
    CTX_CUDA(ctx, ctx->d_slots.reserve(K * slot + 16));
    CTX_CUDA(ctx, ctx->d_in_off.reserve(K)); CTX_CUDA(ctx, ctx->d_out_off.reserve(K)); CTX_CUDA(ctx, ctx->d_in_len.reserve(K));
    CTX_CUDA(ctx, ctx->d_out_cap.reserve(K)); CTX_CUDA(ctx, ctx->d_rwant.reserve(K)); CTX_CUDA(ctx, ctx->d_seg_off.reserve(K));
    CTX_CUDA(ctx, ctx->d_off_b.reserve(K)); CTX_CUDA(ctx, ctx->d_gdst.reserve(K)); CTX_CUDA(ctx, ctx->d_glen.reserve(K));
    CTX_CUDA(ctx, ctx->d_pick.reserve(K)); CTX_CUDA(ctx, ctx->d_out_len.reserve(K)); CTX_CUDA(ctx, ctx->d_status.reserve(K));
    fr::RangeItems a{d_index, info.content_len, d_start, d_len, d_out_off, 0, 0, ctx->d_rfirst.p, ctx->d_ritem.p,
                     (uint64_t)(uintptr_t)ctx->d_slots.p - (uint64_t)(uintptr_t)d_out, slot,
                     ctx->d_in_off.p, ctx->d_out_off.p, ctx->d_in_len.p, ctx->d_out_cap.p, ctx->d_rwant.p,
                     ctx->d_seg_off.p, ctx->d_off_b.p, ctx->d_gdst.p, ctx->d_glen.p, ctx->d_pick.p};
    for (uint32_t r0 = 0; r0 < nr; r0 += kRangeChunk) {
        const uint32_t rc = std::min(kRangeChunk, nr - r0);
        fr::range_plan_kernel<<<(rc + 127) / 128, 128, 0, s>>>(d_index, nb, info.content_len, d_start, d_len, d_written,
                                                               r0, rc, ctx->d_rfirst.p, ctx->d_rcount.p);
        scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_rcount.p, ctx->d_ritem.p, rc);
        CTX_CUDA(ctx, cudaGetLastError());
        uint64_t total = 0;
        CTX_CUDA(ctx, cudaMemcpyAsync(&total, ctx->d_ritem.p + rc, sizeof total, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
        ctx->last_range_blocks += total;
        a.r0 = r0;
        a.rc = rc;
        for (uint64_t j0 = 0; j0 < total; j0 += K) {
            const uint32_t k = (uint32_t)std::min<uint64_t>(K, total - j0), grid = (k + 127) / 128;
            fr::range_items_kernel<<<grid, 128, 0, s>>>(a, j0, k);
            CTX_CUDA(ctx, cudaGetLastError());
            BatchArgs b{d_in, ctx->d_in_off.p, ctx->d_in_len.p, nullptr, d_out, ctx->d_out_off.p, ctx->d_out_cap.p,
                        ctx->d_out_len.p, ctx->d_status.p, nullptr, k, nullptr};
            const lz4b200_status st = launch_decompress(ctx, b, s);
            if (st != LZ4B200_OK) return st;
            fr::range_check_kernel<<<grid, 128, 0, s>>>(ctx->d_rwant.p, ctx->d_out_len.p, ctx->d_status.p, k, ctx->d_bad.p);
            GatherArgs g{ctx->d_slots.p, d_in, ctx->d_seg_off.p, ctx->d_off_b.p, ctx->d_glen.p, ctx->d_glen.p,
                         ctx->d_pick.p, nullptr, d_out, ctx->d_gdst.p, k};
            gather_segments_kernel<<<std::min<uint32_t>(k, (uint32_t)ctx->sm_count * 8), 256, 0, s>>>(g);
            CTX_CUDA(ctx, cudaGetLastError());
        }
    }
    return LZ4B200_OK;
}

// Linked blocks: segments of consecutive touched blocks, each with a look-back of the blocks that hold the 64 KiB of
// content before it.  A round marker-decodes every active segment's blocks (look-back included) in windows of entries
// that fit the frame budget, resolves them and copies the ranges out; a segment with a requested byte still unresolved
// doubles its look-back (in blocks) for the next round, and segments whose look-backs meet merge.  A segment that starts
// at block 0 always resolves: a byte that copies content before byte 0 fails its block.
struct LinkedSeg {
    uint32_t j, a, b;                         // decoded blocks [j, b]; the ranges touch blocks [a, b]
};

lz4b200_status decode_ranges_linked(lz4b200_ctx *ctx, cudaStream_t s, const uint8_t *d_in,
                                    const lz4b200_frame_index_info &info, const lz4b200_frame_index_entry *d_index,
                                    const uint64_t *d_start, const uint64_t *d_len, uint8_t *d_out,
                                    const uint64_t *d_out_off, uint64_t *d_written, uint32_t nr)
{
    const uint32_t nb = (uint32_t)info.nblocks;
    CTX_CUDA(ctx, ctx->d_rtouch.reserve(nb + 1));
    CTX_CUDA(ctx, cudaMemsetAsync(ctx->d_rtouch.p, 0, (nb + 1) * sizeof(int32_t), s));
    fr::range_touch_kernel<<<(nr + 127) / 128, 128, 0, s>>>(d_index, nb, info.content_len, d_start, d_len, d_written, nr,
                                                            ctx->d_rtouch.p);
    CTX_CUDA(ctx, cudaGetLastError());
    std::vector<int32_t> touch(nb + 1);
    std::vector<lz4b200_frame_index_entry> ent(nb);
    CTX_CUDA(ctx, cudaMemcpyAsync(touch.data(), ctx->d_rtouch.p, (nb + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaMemcpyAsync(ent.data(), d_index, nb * sizeof(lz4b200_frame_index_entry), cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaStreamSynchronize(s));
    // the last block whose decoded offset is at most x, as fr::block_at finds it
    auto block_at = [&](uint64_t x) {
        uint32_t lo = 0, hi = nb;
        while (hi - lo > 1) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (ent[mid].decoded_off <= x) lo = mid; else hi = mid;
        }
        return lo;
    };
    std::vector<LinkedSeg> act;
    int32_t run = 0;
    for (uint32_t b = 0; b < nb; b++) {
        run += touch[b];
        if (run <= 0) continue;
        if (!act.empty() && act.back().b + 1 == b) { act.back().b = b; continue; }
        const uint64_t d = ent[b].decoded_off;
        act.push_back({d > fr::kCarry ? block_at(d - fr::kCarry) : 0u, b, b});
    }
    const uint64_t window = std::min<uint64_t>(std::max<uint64_t>(ctx->frame_budget / 4, fr::kCarry + info.block_size),
                                               1u << 30);
    const uint32_t sms = (uint32_t)ctx->sm_count;
    CTX_CUDA(ctx, ctx->d_rcarry.reserve(fr::kCarry));
    uint64_t decodes = 0;
    ctx->last_range_blocks = 0;
    std::vector<fr::MarkBlock> blk;
    std::vector<fr::MarkPiece> piece;
    struct Win { uint32_t blk0, blk1, p0, p1; uint64_t entries; };
    std::vector<Win> wins;
    while (!act.empty()) {
        std::vector<LinkedSeg> m;                                  // merge segments whose look-backs meet
        for (const LinkedSeg &g : act) {
            if (!m.empty() && g.j <= m.back().b + 1) { m.back().j = std::min(m.back().j, g.j); m.back().b = g.b; }
            else m.push_back(g);
        }
        act.swap(m);
        // the round's windows: each segment's blocks in order, a piece per segment and window
        blk.clear(); piece.clear(); wins.clear();
        uint64_t used = 0;
        wins.push_back({0, 0, 0, 0, 0});
        for (uint32_t g = 0; g < act.size(); g++) {
            bool carried = false;
            for (uint32_t k = act[g].j; k <= act[g].b;) {
                if (used && used + fr::kCarry + ent[k].decoded_len > window) {   // a new window
                    wins.back().blk1 = (uint32_t)blk.size(); wins.back().p1 = (uint32_t)piece.size();
                    wins.back().entries = used;
                    wins.push_back({(uint32_t)blk.size(), 0, (uint32_t)piece.size(), 0, 0});
                    used = 0;
                }
                fr::MarkPiece p{ent[k].decoded_off, ent[k].decoded_off, ent[act[g].a].decoded_off, (uint32_t)blk.size(),
                                0, (uint32_t)used, g, carried ? 1u : 0u, 0};
                used += fr::kCarry;
                do {
                    blk.push_back({ent[k].payload_off, ent[k].decoded_off, ent[k].word, ent[k].decoded_len, (uint32_t)used});
                    used += ent[k].decoded_len;
                    p.c1 += ent[k].decoded_len;
                    k++;
                } while (k <= act[g].b && used + ent[k].decoded_len <= window);
                p.blk1 = (uint32_t)blk.size();
                piece.push_back(p);
                carried = true;
            }
        }
        wins.back().blk1 = (uint32_t)blk.size(); wins.back().p1 = (uint32_t)piece.size(); wins.back().entries = used;
        uint64_t most = 0;
        for (const Win &w : wins) most = std::max(most, w.entries);
        CTX_CUDA(ctx, ctx->d_rent.reserve(most));
        CTX_CUDA(ctx, ctx->d_rblk.reserve(blk.size())); CTX_CUDA(ctx, ctx->d_rpiece.reserve(piece.size()));
        CTX_CUDA(ctx, ctx->d_rflag.reserve(act.size()));
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_rblk.p, blk.data(), blk.size() * sizeof(fr::MarkBlock), cudaMemcpyHostToDevice, s));
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_rpiece.p, piece.data(), piece.size() * sizeof(fr::MarkPiece), cudaMemcpyHostToDevice, s));
        CTX_CUDA(ctx, cudaMemsetAsync(ctx->d_rflag.p, 0, act.size() * sizeof(uint32_t), s));
        for (const Win &w : wins) {
            const uint32_t k = w.blk1 - w.blk0, np = w.p1 - w.p0;
            fr::marker_decode_kernel<32><<<(k + 3) / 4, 128, 0, s>>>(d_in, ctx->d_rblk.p + w.blk0, k, ctx->d_rent.p,
                                                                    ctx->d_bad.p);
            fr::resolve_tails_kernel<<<np, 1024, 0, s>>>(ctx->d_rblk.p, ctx->d_rpiece.p + w.p0, ctx->d_rcarry.p,
                                                         ctx->d_rent.p);
            fr::entries_out_kernel<<<std::min<uint32_t>(nr, sms * 8), 256, 0, s>>>(
                ctx->d_rent.p, ctx->d_rpiece.p + w.p0, np, d_start, d_len, info.content_len, d_out, d_out_off, nr,
                ctx->d_rflag.p);
            CTX_CUDA(ctx, cudaGetLastError());
            const fr::MarkPiece &last = piece[w.p1 - 1];           // a segment cut here carries its last 64 KiB on
            if (w.p1 < piece.size() && piece[w.p1].carried)
                CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_rcarry.p, ctx->d_rent.p + last.base + (last.c1 - last.c0),
                                              fr::kCarry * sizeof(uint32_t), cudaMemcpyDeviceToDevice, s));
            decodes += k;
        }
        std::vector<uint32_t> flag(act.size());
        uint32_t bad = 0;
        CTX_CUDA(ctx, cudaMemcpyAsync(flag.data(), ctx->d_rflag.p, act.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaMemcpyAsync(&bad, ctx->d_bad.p, 4, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
        ctx->last_range_blocks = decodes;
        if (bad) return LZ4B200_FRAME_DECOMPRESSION_ERROR;
        m.clear();
        for (uint32_t g = 0; g < act.size(); g++) {
            if (!flag[g]) continue;
            const LinkedSeg &x = act[g];
            if (x.j == 0) return LZ4B200_FRAME_DECOMPRESSION_ERROR;   // cannot happen: such bytes fail their block
            const uint32_t back = 2 * (x.a - x.j);
            m.push_back({back >= x.a ? 0u : x.a - back, x.a, x.b});
        }
        act.swap(m);
    }
    return LZ4B200_OK;
}

}  // namespace

lz4b200_status lz4b200_frame_decompress_ranges_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t n,
                                                      const lz4b200_frame_index_info *info,
                                                      const lz4b200_frame_index_entry *d_index,
                                                      const uint64_t *d_start, const uint64_t *d_len, uint8_t *d_out,
                                                      const uint64_t *d_out_off, uint64_t *d_written, size_t nranges,
                                                      void *stream)
{
    if (!ctx || !info || (!d_in && n) || nranges > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nranges && (!d_start || !d_len || !d_out || !d_out_off || !d_written)) return LZ4B200_INVALID_ARGUMENT;
    ctx->last_range_blocks = 0;
    // the info is checked before anything of the index is read: a block size the format allows, a block count the
    // planner can index, a content length the blocks can hold
    const uint64_t bs = info->block_size, nbx = info->nblocks;
    const bool bs_ok = bs == (64u << 10) || bs == (256u << 10) || bs == (1u << 20) || bs == (4u << 20) || bs == (8u << 20);
    if (nbx >= 0xffffffffull || (nbx && (!d_index || !bs_ok)) || info->content_len > nbx * bs)
        return LZ4B200_INVALID_ARGUMENT;
    if (!nranges) return LZ4B200_OK;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nb = (uint32_t)nbx, nr = (uint32_t)nranges;
    CTX_CUDA(ctx, ctx->d_bad.reserve(1));
    CTX_CUDA(ctx, cudaMemsetAsync(ctx->d_bad.p, 0, 4, s));
    uint32_t bad = 0;
    if (nb) {
        fr::index_check_kernel<<<(nb + 255) / 256, 256, 0, s>>>(d_index, nb, n, bs, info->content_len, ctx->d_bad.p);
        CTX_CUDA(ctx, cudaGetLastError());
        CTX_CUDA(ctx, cudaMemcpyAsync(&bad, ctx->d_bad.p, 4, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
        if (bad) return LZ4B200_INVALID_ARGUMENT;
    }
    const lz4b200_status st = info->linked
        ? decode_ranges_linked(ctx, s, d_in, *info, d_index, d_start, d_len, d_out, d_out_off, d_written, nr)
        : decode_ranges_independent(ctx, s, d_in, *info, d_index, d_start, d_len, d_out, d_out_off, d_written, nr);
    if (st == LZ4B200_CUDA_ERROR) return st;
    CTX_CUDA(ctx, cudaMemcpyAsync(&bad, ctx->d_bad.p, 4, cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaStreamSynchronize(s));
    if (st != LZ4B200_OK) return st;
    return bad ? LZ4B200_FRAME_DECOMPRESSION_ERROR : LZ4B200_OK;
}

uint64_t lz4b200_ctx_last_range_blocks(const lz4b200_ctx *ctx)
{
    return ctx ? ctx->last_range_blocks : 0;
}

size_t lz4b200_ctx_device_bytes(const lz4b200_ctx *ctx)
{
    if (!ctx) return 0;
    size_t b = 0;
    auto add = [&b](const auto &buf) { b += buf.cap * sizeof(*buf.p); };
    add(ctx->d_tickets); add(ctx->d_gtab16);
#ifdef LZ4B200_AB_VARIANTS
    add(ctx->d_ttab16); add(ctx->d_gtag32);
#endif
    add(ctx->d_in); add(ctx->d_out); add(ctx->d_slots); add(ctx->d_flags); add(ctx->d_pick); add(ctx->d_dict);
    add(ctx->d_in_off); add(ctx->d_out_off); add(ctx->d_seg_off); add(ctx->d_expected); add(ctx->d_off_b);
    add(ctx->d_in_len); add(ctx->d_out_cap); add(ctx->d_out_len); add(ctx->d_info); add(ctx->d_seg_size);
    add(ctx->d_payload_len); add(ctx->d_link_first); add(ctx->d_stored_len); add(ctx->d_done);
    add(ctx->d_status); add(ctx->d_walk); add(ctx->d_desc); add(ctx->d_bad); add(ctx->d_content); add(ctx->d_result);
    add(ctx->d_fwalk); add(ctx->d_fcount); add(ctx->d_fnb); add(ctx->d_bframe);
    add(ctx->d_bslot); add(ctx->d_glen); add(ctx->d_fscan); add(ctx->d_gdst); add(ctx->d_fhash); add(ctx->d_fplan);
    add(ctx->d_gframe); add(ctx->d_reach); add(ctx->d_rfirst); add(ctx->d_rcount); add(ctx->d_rwant); add(ctx->d_ritem);
    add(ctx->d_rtouch); add(ctx->d_rent); add(ctx->d_rcarry); add(ctx->d_rflag); add(ctx->d_rblk); add(ctx->d_rpiece);
    if (const Pipeline *p = ctx->pipe.get()) {
        for (const Lane &l : p->lane) { add(l.in); add(l.slots); add(l.out); }
        add(p->d_tickets);
    }
    return b;
}

// ---- streaming frame decoder (FrameDecoder over device memory, frame/decompress.rs:109-342) ------------------------------
// The decoder holds what must outlive a call: the walk of the frame in progress, the frame's output so far, a linked
// frame's window and the running content hash.  Descriptors, slots and staged payload are the context's scratch, so other
// calls on the context may come between two of its calls.
struct lz4b200_frame_decoder {
    lz4b200_ctx *ctx = nullptr;
    int device = 0;                           // the context's device (the decoder's buffers live there)
    fw::FrameWalk w;                          // the frame in progress, offsets from its first byte (fresh: no frame yet)
    uint64_t written = 0;                     // bytes the frame has decoded so far
    uint32_t win_len = 0, win = 0;            // linked frames: bytes in the window, and which half of d_win holds them
    DevBuf<uint8_t> d_win;                    // two halves of kWindowBytes: the window, and the next one
    DevBuf<lz4b200_xxh32_state> d_content;    // the running content hash
    DevBuf<uint64_t> d_need;                  // what the walk needs to go on
};

namespace {

// The frame ends in this call with status `st` after `consumed` bytes; the decoder waits for the next frame.
void decoder_finish(lz4b200_frame_decoder *dec, lz4b200_frame_decoder_step &step, lz4b200_status st, uint64_t consumed)
{
    step.frame_done = 1;
    step.result.status = st;
    step.result.consumed = consumed;
    step.result.written = dec->written;
    dec->w = fw::FrameWalk{};
    dec->written = 0;
    dec->win_len = 0;
}

// One call: walk the presented chunk, take the blocks that fit out_cap and the frame budget, check their checksums,
// decode them as one group of the group loop, and carry the window and the content hash to the next call.
lz4b200_status decoder_step(lz4b200_frame_decoder *dec, cudaStream_t s, const uint8_t *d_in, size_t n, bool eof,
                            uint8_t *d_out, size_t out_cap, lz4b200_frame_decoder_step &step)
{
    lz4b200_ctx *ctx = dec->ctx;
    const fw::FrameWalk w0 = dec->w;
    const uint64_t at = w0.ip;                                    // the frame's bytes before d_in[0]
    CTX_CUDA(ctx, ctx->d_walk.reserve(2)); CTX_CUDA(ctx, ctx->d_desc.reserve(kDeviceWalkChunk));
    CTX_CUDA(ctx, ctx->d_bad.reserve(1));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_walk.p, &w0, sizeof w0, cudaMemcpyHostToDevice, s));
    frame_walk_stream_kernel<<<1, 1, 0, s>>>(d_in, n, eof, ctx->d_walk.p, ctx->d_desc.p, kDeviceWalkChunk, dec->d_need.p);
    CTX_CUDA(ctx, cudaGetLastError());
    fw::FrameWalk w1;
    uint64_t need = 0;
    CTX_CUDA(ctx, cudaMemcpyAsync(&w1, ctx->d_walk.p, sizeof w1, cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaMemcpyAsync(&need, dec->d_need.p, sizeof need, cudaMemcpyDeviceToHost, s));
    CTX_CUDA(ctx, cudaStreamSynchronize(s));
    const uint32_t k = (uint32_t)(w1.nblocks - w0.nblocks);
    std::vector<fw::FrameBlockDesc> blocks(k);                    // payload offsets from d_in[0]
    if (k) {
        CTX_CUDA(ctx, cudaMemcpyAsync(blocks.data(), ctx->d_desc.p, k * sizeof(fw::FrameBlockDesc), cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
    }

    // the blocks this call decodes: the longest prefix whose decoded bounds fit out_cap and that the group loop would
    // not cut (slots and input span within the frame budget)
    uint32_t t = 0;
    for (uint64_t bound = 0, slots = 0; t < k; t++) {
        const fw::FrameBlockDesc &b = blocks[t];
        const uint64_t cap = fw::block_slot_cap(b, w1.bs);
        const uint64_t ob = fw::block_stored(b) ? fw::block_len(b) : cap;
        if (bound + ob > out_cap) break;
        if (t && fw::group_cut(slots, cap, b.payload_off + fw::block_len(b) - blocks[0].payload_off, ctx->frame_budget))
            break;
        bound += ob;
        slots += fw::slot_bytes(cap);
    }
    if (k && !t) return LZ4B200_FRAME_OUTPUT_FULL;                // the next block alone does not fit: nothing is taken

    // block checksums of the blocks taken: the first that fails ends the frame there
    uint32_t bad = fw::kNoBlock;
    if (t && (w1.flg & 0x10)) {
        fw::FrameWalk wt = w1;
        wt.nblocks = t;
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_walk.p + 1, &wt, sizeof wt, cudaMemcpyHostToDevice, s));
        CTX_CUDA(ctx, cudaMemsetAsync(ctx->d_bad.p, 0xff, 4, s));
        block_checksum_kernel<<<(t + 127) / 128, 128, 0, s>>>(d_in, ctx->d_desc.p, ctx->d_walk.p + 1, 0, ctx->d_bad.p);
        CTX_CUDA(ctx, cudaGetLastError());
        CTX_CUDA(ctx, cudaMemcpyAsync(&bad, ctx->d_bad.p, 4, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
    }
    fw::FrameWalk wn = w1;                                        // the walk as this call leaves it
    if (bad < t) {
        fw::frame_walk_fail_block(wn, blocks[bad], (uint32_t)(w0.nblocks + bad));
        wn.ip += at;
        wn.stage = fw::kWalkDone;
        t = bad;
    } else if (t < k) {
        wn.ip = at + blocks[t].payload_off - 4;                   // at the BlockInfo of the first block not taken
        wn.nblocks = w0.nblocks + t;
        wn.stage = fw::kWalkBlocks;
        wn.status = LZ4B200_OK;
        wn.closed = wn.has_checksum = 0;
        wn.content_checksum = 0;
        need = 0;
    }
    blocks.resize(t);
    lz4b200_frame_result r;
    uint32_t failed = fw::kNoBlock;
    const lz4b200_status st = decode_frame_blocks(ctx, s, true, d_in, d_out, out_cap, wn, blocks,
                                                  wn.stage == fw::kWalkDone, dec->written, dec->d_content.p, &r, nullptr,
                                                  dec->d_win.p + (size_t)dec->win * kWindowBytes, dec->win_len, &failed);
    if (st != LZ4B200_OK) return st;
    if (r.status == LZ4B200_FRAME_OUTPUT_FULL) return LZ4B200_FRAME_OUTPUT_FULL;
    const uint64_t got = r.written - dec->written;
    dec->written = r.written;
    step.written = got;
    if (r.status == LZ4B200_FRAME_DECOMPRESSION_ERROR) {
        // the reference's reader stands after the failing block and its checksum
        const fw::FrameBlockDesc &b = blocks[failed];
        step.consumed = b.payload_off + fw::block_len(b) + ((wn.flg & 0x10) ? 4 : 0);
        step.result = r;
        decoder_finish(dec, step, LZ4B200_FRAME_DECOMPRESSION_ERROR, at + step.consumed);
        return LZ4B200_OK;
    }
    step.consumed = wn.ip - at;
    if (wn.stage == fw::kWalkDone) {
        step.result = r;
        decoder_finish(dec, step, (lz4b200_status)r.status, wn.ip);
        return LZ4B200_OK;
    }
    if (wn.linked && got) {
        uint8_t *old = dec->d_win.p + (size_t)dec->win * kWindowBytes;
        uint8_t *next = dec->d_win.p + (size_t)(dec->win ^ 1) * kWindowBytes;
        window_update_kernel<<<64, 256, 0, s>>>(old, dec->win_len, d_out, got, next);
        CTX_CUDA(ctx, cudaGetLastError());
        dec->win ^= 1;
        dec->win_len = (uint32_t)std::min<uint64_t>(kWindowBytes, dec->win_len + got);
    }
    dec->w = wn;
    step.need = need;
    return LZ4B200_OK;
}

}  // namespace

lz4b200_status lz4b200_frame_decoder_create(lz4b200_ctx *ctx, lz4b200_frame_decoder **out)
{
    if (!ctx || !out) return LZ4B200_INVALID_ARGUMENT;
    *out = nullptr;
    DeviceGuard guard(ctx->device);
    lz4b200_frame_decoder *dec = new lz4b200_frame_decoder();
    dec->ctx = ctx;
    dec->device = ctx->device;
    if (!ctx->check(dec->d_win.reserve(2 * kWindowBytes), "decoder window") ||
        !ctx->check(dec->d_content.reserve(1), "decoder content hash") || !ctx->check(dec->d_need.reserve(1), "decoder need")) {
        delete dec;
        return LZ4B200_CUDA_ERROR;
    }
    *out = dec;
    return LZ4B200_OK;
}

void lz4b200_frame_decoder_destroy(lz4b200_frame_decoder *dec)
{
    if (!dec) return;
    DeviceGuard guard(dec->device);
    delete dec;
}

lz4b200_status lz4b200_frame_decoder_decode_device(lz4b200_frame_decoder *dec, const uint8_t *d_in, size_t n,
                                                   int end_of_input, uint8_t *d_out, size_t out_cap,
                                                   lz4b200_frame_decoder_step *step, void *stream)
{
    if (!dec || !step || (!d_in && n) || (!d_out && out_cap)) return LZ4B200_INVALID_ARGUMENT;
    *step = lz4b200_frame_decoder_step{};
    lz4b200_ctx *ctx = dec->ctx;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    const lz4b200_status st = decoder_step(dec, s, d_in, n, end_of_input != 0, d_out, out_cap, *step);
    if (st != LZ4B200_CUDA_ERROR) CTX_CUDA(ctx, cudaStreamSynchronize(s));
    return st;
}

// ---- streaming frame encoder (FrameEncoder over device memory, frame/compress.rs:62-404) -------------------------------
// The encoder holds what must outlive a call: the stream state of fe::State, the input buffer of one group of whole
// blocks, the running content hash and the output position of the call.  Descriptors and slots are the context's
// scratch, so other calls on the context may come between two of its calls.
struct lz4b200_frame_encoder {
    lz4b200_ctx *ctx = nullptr;
    int device = 0;
    lz4b200_frame_info info{};                // as created; the block size resolves into st
    fe::State st;
    DevBuf<uint8_t> d_buf;                    // the input buffer: st.group blocks of the open frame's block size
    DevBuf<lz4b200_xxh32_state> d_content;    // the running content hash
    DevBuf<uint64_t> d_pos;                   // the call's output position, double-buffered: group g moves it from
                                              // d_pos[g % 2] to d_pos[(g + 1) % 2]
};

lz4b200_status lz4b200_frame_encoder_create(lz4b200_ctx *ctx, const lz4b200_frame_info *info, lz4b200_frame_encoder **out)
{
    if (!ctx || !info || !out) return LZ4B200_INVALID_ARGUMENT;
    *out = nullptr;
    if (info->linked) return LZ4B200_FRAME_LINKED_UNSUPPORTED;
    const int id = info->block_size_id;
    if (id != 0 && (id < 4 || id > 7)) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    lz4b200_frame_encoder *enc = new lz4b200_frame_encoder();
    enc->ctx = ctx;
    enc->device = ctx->device;
    enc->info = *info;
    enc->st.block_size_id = id;
    if (!ctx->check(enc->d_content.reserve(1), "encoder content hash") || !ctx->check(enc->d_pos.reserve(2), "encoder position")) {
        delete enc;
        return LZ4B200_CUDA_ERROR;
    }
    *out = enc;
    return LZ4B200_OK;
}

void lz4b200_frame_encoder_destroy(lz4b200_frame_encoder *enc)
{
    if (!enc) return;
    DeviceGuard guard(enc->device);
    delete enc;
}

size_t lz4b200_frame_encoder_bound(const lz4b200_frame_encoder *enc, size_t n, int op)
{
    if (!enc || op < fe::kWrite || op > fe::kFinish) return 0;
    return fe::call_bound(enc->st, enc->info, enc->ctx->frame_budget, n, op);
}

uint64_t lz4b200_frame_encoder_content_len(const lz4b200_frame_encoder *enc) { return enc ? enc->st.content_len : 0; }

// One call: plan it on the host (fe::plan_call), then enqueue the header, per step the copy into the buffer, the
// group's plan through compress_frames at the call's position and its content hash, and the tail.  Only kernel
// arguments cross PCIe.
lz4b200_status lz4b200_frame_encoder_encode_device(lz4b200_frame_encoder *enc, const uint8_t *d_in, size_t n, int op,
                                                   uint8_t *d_out, size_t out_cap, uint64_t *d_written, void *stream)
{
    if (!enc || !d_written || (!d_out && out_cap)) return LZ4B200_INVALID_ARGUMENT;
    if (!d_in && n) return LZ4B200_INVALID_ARGUMENT;
    if (op < fe::kWrite || op > fe::kFinish) return LZ4B200_INVALID_ARGUMENT;
    lz4b200_ctx *ctx = enc->ctx;
    if (out_cap < fe::call_bound(enc->st, enc->info, ctx->frame_budget, n, op)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    const fe::CallPlan p = fe::plan_call(enc->st, enc->info, ctx->frame_budget, n, op);
    const size_t bs = fe::block_bytes(p.block_size_id);
    const size_t want = p.group * bs;
    if (p.header && want != enc->d_buf.cap)                  // the buffer follows the block size and the budget
        CTX_CUDA(ctx, enc->d_buf.resize(want));

    lz4b200_frame_info info = enc->info;
    info.block_size_id = p.block_size_id;
    FrameHeaderBytes hdr{};
    if (p.header) hdr.len = (uint8_t)lz4b200_frame_write_header(&info, hdr.b, sizeof hdr.b);
    uint64_t *pos = enc->d_pos.p;
    encoder_head_kernel<<<1, 1, 0, s>>>(d_out, hdr, pos);
    CTX_CUDA(ctx, cudaGetLastError());
    if (p.header && info.content_checksum) {                 // a new frame's content hash (compress.rs:253)
        xxh32_reset_kernel<<<1, 1, 0, s>>>(enc->d_content.p, 0);
        CTX_CUDA(ctx, cudaGetLastError());
    }
    uint32_t g = 0;                                          // groups so far: the position is at pos[g % 2]
    for (const fe::Step &st : p.steps) {
        if (st.len)
            CTX_CUDA(ctx, cudaMemcpyAsync(enc->d_buf.p + st.dst, d_in + st.src, st.len, cudaMemcpyDeviceToDevice, s));
        if (!st.group_len) continue;
        const fb::FramePlan plan = fe::group_plan(st, bs);
        const lz4b200_status r = compress_frames(ctx, enc->d_buf.p, &plan, 1,
                                                 (uint32_t)std::min<uint64_t>(st.group_len, bs), info.block_checksums,
                                                 false, d_out, nullptr, pos + g % 2, pos + (g + 1) % 2, s);
        if (r != LZ4B200_OK) return r;
        g++;
        if (info.content_checksum) {                          // compress.rs:319-321, in stream order
            content_hash_kernel<<<1, 256, 0, s>>>(enc->d_content.p, enc->d_buf.p, st.group_len);
            CTX_CUDA(ctx, cudaGetLastError());
        }
    }
    encoder_tail_kernel<<<1, 1, 0, s>>>(d_out, pos + g % 2, p.endmark != 0, info.content_checksum ? enc->d_content.p : nullptr,
                                        d_written);
    CTX_CUDA(ctx, cudaGetLastError());
    enc->st = p.next;
    return (lz4b200_status)p.status;
}

}  // extern "C"
