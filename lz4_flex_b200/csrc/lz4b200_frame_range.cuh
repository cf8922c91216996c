// lz4b200_frame_range.cuh — random access into an LZ4 frame in device memory: the block sizing kernel behind
// lz4b200_frame_index_device and the planning kernels of lz4b200_frame_decompress_ranges_device.
//
// A frame does not record how many bytes a block decodes to.  The sizing walk follows a block's token stream without
// writing anything: literal runs are skipped, matches only advance the output position.  It makes every check the
// block decoder (lz4_decompress_blocks / _linked) makes, in the same order, so its (length, status, expected) are the
// decoder's for the same block and capacity.  One thread per block: the walk is one dependent chain of byte loads,
// and with no copies there is nothing for more lanes to share.
#pragma once
#include <stdint.h>

#include "../../include/lz4b200.h"
#include "lz4b200_frame_walk.cuh"

namespace lz4b200 {
namespace fr {

struct SizeResult {
    uint32_t len;        // decoded bytes (status OK)
    int32_t status;
    uint64_t expected;   // OutputTooSmall{expected}
    uint32_t reach;      // linked blocks: how far the deepest offset so far reached before the block's first byte
};

// The checked decode loop (decode_sequence_checked, decompress.rs:330-444) with the copies left out.  An offset that
// reaches before the block is OffsetOutOfBounds in an independent block; in a linked block its depth is recorded at
// the point the decoder checks it (after the match length, before the capacity), and the caller decides it once the
// block's decoded offset in the frame is known.
__device__ __forceinline__ SizeResult size_block(const uint8_t *__restrict__ src, uint32_t n, uint32_t cap, bool linked)
{
    SizeResult r{0u, LZ4B200_OK, 0ull, 0u};
    if (n == 0) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }   // decompress.rs:207-209
    uint32_t ip = 0, op = 0;
    for (;;) {
        const uint32_t tok = __ldg(src + ip++);
        uint64_t lit = tok >> 4;
        if (lit == 15) {
            for (;;) {
                if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }
                const uint32_t b = __ldg(src + ip++);
                lit += b;
                if (b != 255) break;
            }
        }
        if (lit) {
            if (lit > (uint64_t)(n - ip)) { r.status = LZ4B200_DEC_LITERAL_OUT_OF_BOUNDS; return r; }
            if (lit > (uint64_t)(cap - op)) { r.status = LZ4B200_DEC_OUTPUT_TOO_SMALL; r.expected = (uint64_t)op + lit; return r; }
            ip += (uint32_t)lit; op += (uint32_t)lit;
        }
        if (ip >= n) break;                                        // the stream ends after literals
        if (n - ip < 2) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }
        const uint32_t dist = (uint32_t)__ldg(src + ip) | ((uint32_t)__ldg(src + ip + 1) << 8);
        ip += 2;
        if (dist == 0) { r.status = LZ4B200_DEC_OFFSET_ZERO; return r; }
        uint64_t mlen = 4u + (tok & 15u);
        if (mlen == 19) {
            for (;;) {
                if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }
                const uint32_t b = __ldg(src + ip++);
                mlen += b;
                if (b != 255) break;
            }
        }
        if (dist > op) {
            if (!linked) { r.status = LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS; return r; }
            r.reach = max(r.reach, dist - op);
        }
        if (mlen > (uint64_t)(cap - op)) { r.status = LZ4B200_DEC_OUTPUT_TOO_SMALL; r.expected = (uint64_t)op + mlen; return r; }
        op += (uint32_t)mlen;
        if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }   // may not end on a match
    }
    r.len = op;
    return r;
}

// One thread per block of the walk: its decoded length, status, OutputTooSmall expected and capacity (the frame
// decoders' out_cap, min(block size, 255 x payload)), and a linked block's reach.  A stored block is its payload.
__global__ void __launch_bounds__(128) block_size_kernel(const uint8_t *in, const fw::FrameBlockDesc *desc, uint32_t nb,
                                                         uint64_t bs, bool linked, uint32_t *len, int32_t *status,
                                                         uint64_t *expected, uint32_t *cap, uint32_t *reach)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const fw::FrameBlockDesc d = desc[b];
    SizeResult r{fw::block_len(d), LZ4B200_OK, 0ull, 0u};
    const uint32_t c = fw::block_stored(d) ? 0u : (uint32_t)fw::block_decoded_cap(fw::block_len(d), bs);
    if (!fw::block_stored(d)) r = size_block(in + d.payload_off, fw::block_len(d), c, linked);
    len[b] = r.status == LZ4B200_OK ? r.len : 0u;
    status[b] = r.status;
    expected[b] = r.expected;
    cap[b] = c;
    reach[b] = r.reach;
}

// Linked frames, once the decoded offsets are known (off: the exclusive scan of len): a block whose offsets reach
// further back than the frame's output before it is OffsetOutOfBounds.  Only the blocks of the frame's first 64 KiB can
// fail here (an offset is at most 65 535).  The reach only counts offsets checked before the walk stopped, so an
// offset out of bounds comes before any error the walk met, as in the decoder.  The offsets of blocks after the first
// failing one are not theirs, but the frame ends at that block anyway.
__global__ void __launch_bounds__(128) block_reach_kernel(const uint64_t *off, const uint32_t *reach, uint32_t nb,
                                                          int32_t *status, uint64_t *expected, uint32_t *len)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb || reach[b] <= off[b]) return;
    status[b] = LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS;
    expected[b] = 0;
    len[b] = 0;
}

// The index entries of the delivered blocks: decoded offset and length as the frame's result step laid them out.
__global__ void __launch_bounds__(128) index_entries_kernel(const fw::FrameBlockDesc *desc, const uint64_t *dst_off,
                                                            const uint32_t *glen, uint32_t nb,
                                                            lz4b200_frame_index_entry *index)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    index[b] = lz4b200_frame_index_entry{desc[b].payload_off, dst_off[b], desc[b].word, glen[b]};
}

// ---- range decode ---------------------------------------------------------------------------------------------------
// The index comes from outside the library: every entry is checked before any is used.  Payloads lie inside the
// n input bytes and are at most a block; decoded lengths are at most a block (a stored block's is its payload); decoded
// offsets are the running sum of the lengths and end at content_len.  *bad receives 1 when an entry fails.
__global__ void __launch_bounds__(256) index_check_kernel(const lz4b200_frame_index_entry *index, uint32_t nb, uint64_t n,
                                                          uint64_t bs, uint64_t content_len, uint32_t *bad)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const lz4b200_frame_index_entry e = index[b];
    const uint64_t plen = e.word & 0x7fffffffu;
    const bool stored = (e.word & 0x80000000u) != 0;
    bool ok = e.payload_off <= n && plen <= n - e.payload_off && plen <= bs && e.decoded_len <= bs &&
              (!stored || e.decoded_len == plen);
    ok = ok && (b == 0 ? e.decoded_off == 0 : e.decoded_off == index[b - 1].decoded_off + index[b - 1].decoded_len);
    if (b == nb - 1) ok = ok && e.decoded_off <= content_len && e.decoded_len == content_len - e.decoded_off;
    if (!ok) atomicOr(bad, 1u);
}

// The last block whose decoded offset is at most x (entries checked, so offsets ascend; block 0 is at 0).
__device__ __forceinline__ uint32_t block_at(const lz4b200_frame_index_entry *index, uint32_t nb, uint64_t x)
{
    uint32_t lo = 0, hi = nb;                         // index[lo].decoded_off <= x; index[hi].decoded_off > x (hi = nb: none)
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (index[mid].decoded_off <= x) lo = mid; else hi = mid;
    }
    return lo;
}

// A range clipped to the content like a Python slice: [s, e).
__device__ __forceinline__ void clip_range(uint64_t start, uint64_t len, uint64_t content_len, uint64_t &s, uint64_t &e)
{
    s = min(start, content_len);
    e = s + min(len, content_len - s);
}

// One thread per range of the chunk [r0, r0 + rc): its clipped length, its first block and how many blocks it touches.
__global__ void __launch_bounds__(128) range_plan_kernel(const lz4b200_frame_index_entry *index, uint32_t nb,
                                                         uint64_t content_len, const uint64_t *start, const uint64_t *len,
                                                         uint64_t *written, uint32_t r0, uint32_t rc, uint32_t *first,
                                                         uint32_t *count)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rc) return;
    uint64_t s, e;
    clip_range(start[r0 + i], len[r0 + i], content_len, s, e);
    written[r0 + i] = e - s;
    if (e == s) { first[i] = 0; count[i] = 0; return; }
    const uint32_t b0 = block_at(index, nb, s), b1 = block_at(index, nb, e - 1);
    first[i] = b0;
    count[i] = b1 - b0 + 1;
}

// The decode and copy of one (range, block) item of the window [j0, j0 + k), one thread per item (item_off: the
// exclusive scan of the chunk's counts).  A compressed block wholly inside its range decodes into d_out in place, with
// exactly its indexed length as capacity; a partial one into slot j - j0 of the scratch, then its part is copied out; a
// stored block's part is copied from the payload.  Items that decode nothing get in_len 0 and pick 1.
struct RangeItems {
    const lz4b200_frame_index_entry *index;
    uint64_t content_len;
    const uint64_t *start, *len, *out_off;    // the caller's arrays, from range r0
    uint32_t r0, rc;
    const uint32_t *first;
    const uint64_t *item_off;
    uint64_t slot_base;                       // the scratch slots' address minus d_out's (mod 2^64)
    uint64_t slot_bytes;
    // per item: the decoder's arguments, the length the block must decode to, and the copy
    uint64_t *in_off, *dec_off;
    uint32_t *in_len, *dec_cap, *want;
    uint64_t *copy_src_a, *copy_src_b, *copy_dst;
    uint32_t *copy_len;
    uint8_t *pick;
};

__global__ void __launch_bounds__(128) range_items_kernel(RangeItems a, uint64_t j0, uint32_t k)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= k) return;
    const uint64_t j = j0 + t;
    uint32_t lo = 0, hi = a.rc;                       // the range: item_off[lo] <= j < item_off[lo + 1]
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (a.item_off[mid] <= j) lo = mid; else hi = mid;
    }
    const uint32_t r = lo;
    const lz4b200_frame_index_entry e = a.index[a.first[r] + (uint32_t)(j - a.item_off[r])];
    uint64_t s, end;
    clip_range(a.start[a.r0 + r], a.len[a.r0 + r], a.content_len, s, end);
    const uint64_t d0 = e.decoded_off, d1 = d0 + e.decoded_len;
    const uint64_t from = max(s, d0), to = min(end, d1);
    const bool stored = (e.word & 0x80000000u) != 0, whole = from == d0 && to == d1;
    const uint64_t dst = a.out_off[a.r0 + r] + (from - s);
    a.in_off[t] = e.payload_off;
    a.in_len[t] = stored ? 0u : (e.word & 0x7fffffffu);
    a.dec_cap[t] = stored ? 0u : e.decoded_len;
    a.want[t] = stored ? 0xffffffffu : e.decoded_len;
    a.dec_off[t] = whole ? dst : a.slot_base + t * a.slot_bytes;
    a.pick[t] = stored ? 1 : 0;
    a.copy_src_a[t] = t * a.slot_bytes + (from - d0);
    a.copy_src_b[t] = e.payload_off + (from - d0);
    a.copy_dst[t] = dst;
    a.copy_len[t] = stored || !whole ? (uint32_t)(to - from) : 0u;
}

// Every decoded block of the window produced exactly its indexed length: else *bad = 1.
__global__ void __launch_bounds__(128) range_check_kernel(const uint32_t *want, const uint32_t *out_len,
                                                          const int32_t *status, uint32_t k, uint32_t *bad)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= k || want[t] == 0xffffffffu) return;
    if (status[t] != LZ4B200_OK || out_len[t] != want[t]) atomicOr(bad, 1u);
}

// Linked frames: the clipped end of the furthest range, into *end (atomicMax).
__global__ void __launch_bounds__(128) range_end_kernel(const uint64_t *start, const uint64_t *len, uint64_t content_len,
                                                        uint64_t *written, uint32_t nr, unsigned long long *end)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nr) return;
    uint64_t s, e;
    clip_range(start[i], len[i], content_len, s, e);
    written[i] = e - s;
    if (e > s) atomicMax(end, (unsigned long long)e);
}

// Linked frames: every range takes its part of content [g0, g1), decoded at src, one CTA per range at a time.
__global__ void __launch_bounds__(256) range_slice_kernel(const uint8_t *src, uint64_t g0, uint64_t g1,
                                                          const uint64_t *start, const uint64_t *len, uint64_t content_len,
                                                          uint8_t *out, const uint64_t *out_off, uint32_t nr)
{
    for (uint32_t i = blockIdx.x; i < nr; i += gridDim.x) {
        uint64_t s, e;
        clip_range(start[i], len[i], content_len, s, e);
        const uint64_t from = max(s, g0), to = min(e, g1);
        if (from >= to) continue;
        uint8_t *d = out + out_off[i] + (from - s);
        const uint8_t *p = src + (from - g0);
        for (uint64_t x = threadIdx.x; x < to - from; x += blockDim.x) d[x] = p[x];
    }
}

}  // namespace fr
}  // namespace lz4b200
