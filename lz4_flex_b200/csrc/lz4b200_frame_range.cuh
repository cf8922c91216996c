// lz4b200_frame_range.cuh — random access into LZ4 frames in device memory: the block sizing kernel behind
// lz4b200_frame_index_device and _index_batch_device, and the planning kernels of lz4b200_frame_decompress_ranges_device
// and _ranges_batch_device.  The one-frame calls run as calls of one frame.
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
#include "lz4b200_kernels.cuh"

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

// One thread per block of an index group (the GroupFrames of the frame decoders' result step, one per frame): its
// decoded length, status, OutputTooSmall expected and capacity (the frame decoders' out_cap, min(block size, 255 x
// payload)), and a linked block's reach.  The block's frame gives the payload's place, the block size and the block
// mode.  A stored block is its payload.  The group holds nb blocks, or *nb_dev (at most nb) when the count is only known
// on the device.
__global__ void __launch_bounds__(128) block_size_kernel(const uint8_t *in, const fw::FrameBlockDesc *desc,
                                                         const uint32_t *bframe, const GroupFrame *frames, uint32_t nb,
                                                         uint32_t *len, int32_t *status, uint64_t *expected,
                                                         uint32_t *cap, uint32_t *reach, const uint32_t *nb_dev = nullptr)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb || (nb_dev && b >= *nb_dev)) return;
    const GroupFrame &p = frames[bframe[b]];
    const uint64_t bs = p.walk->bs;
    const fw::FrameBlockDesc d = desc[b];
    SizeResult r{fw::block_len(d), LZ4B200_OK, 0ull, 0u};
    const uint32_t c = fw::block_stored(d) ? 0u : (uint32_t)fw::block_decoded_cap(fw::block_len(d), bs);
    if (!fw::block_stored(d)) r = size_block(in + p.in_off + d.payload_off, fw::block_len(d), c, p.walk->linked != 0);
    len[b] = r.status == LZ4B200_OK ? r.len : 0u;
    status[b] = r.status;
    expected[b] = r.expected;
    cap[b] = c;
    reach[b] = r.reach;
}

// Linked frames: a block whose offsets reach further back than the frame's output before it is OffsetOutOfBounds.
// One warp per frame scans the decoded lengths of its blocks from the frame's block 0 (a segmented scan), only over the
// frame's first 64 KiB: an offset is at most 65 535, so no later block can fail here.  The reach only counts offsets
// checked before the walk stopped, so an offset out of bounds comes before any error the walk met, as in the decoder.
// The offsets of blocks after the first failing one are not theirs, but the frame ends at that block anyway.
__global__ void __launch_bounds__(128) frame_reach_kernel(const GroupFrame *frames, uint32_t gn, const uint32_t *reach,
                                                          int32_t *status, uint64_t *expected, uint32_t *len)
{
    const uint32_t g = (blockIdx.x * blockDim.x + threadIdx.x) / 32, lane = threadIdx.x & 31;
    if (g >= gn) return;                                    // whole warps
    const GroupFrame p = frames[g];
    if (!p.walk->linked) return;
    uint64_t total = 0;                                     // the frame's decoded bytes before block k0
    for (uint32_t k0 = 0; k0 < p.nblocks && total < 65536; k0 += 32) {
        const uint32_t k = k0 + lane, b = p.base + k;
        const uint32_t l = k < p.nblocks ? len[b] : 0u;
        uint64_t x = l;
        for (int d = 1; d < 32; d <<= 1) {
            const uint64_t y = __shfl_up_sync(kFull, x, d);
            if (lane >= d) x += y;
        }
        if (k < p.nblocks && reach[b] > total + x - l) {
            status[b] = LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS;
            expected[b] = 0;
            len[b] = 0;
        }
        total += __shfl_sync(kFull, x, 31);
    }
}

// The index entries of the group's blocks: decoded offset and length as the frame's result step laid them out.  Block
// k of frame g goes to index[entry_off[g] + k] (entry_off null: one frame, at index[k]).
__global__ void __launch_bounds__(128) index_entries_kernel(const fw::FrameBlockDesc *desc, const uint32_t *bframe,
                                                            const GroupFrame *frames, const uint64_t *dst_off,
                                                            const uint32_t *glen, uint32_t nb, const uint64_t *entry_off,
                                                            lz4b200_frame_index_entry *index)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const uint32_t g = bframe[b];
    const uint64_t at = (entry_off ? entry_off[g] : 0ull) + (b - frames[g].base);
    index[at] = lz4b200_frame_index_entry{desc[b].payload_off, dst_off[b], desc[b].word, glen[b]};
}

// Each frame's info once the result step ran: its block size and mode from the walk, the blocks delivered (those before
// the first that failed its checksum or its decode) and their decoded total, and the frame's result.
__global__ void __launch_bounds__(128) index_info_kernel(const GroupFrame *frames, uint32_t gn,
                                                         lz4b200_frame_index_info *info)
{
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= gn) return;
    const GroupFrame &p = frames[g];
    lz4b200_frame_index_info i{};
    i.result = *p.result;
    i.block_size = p.walk->bs;
    i.nblocks = min(p.nblocks, p.bad);
    i.content_len = i.result.written;
    i.linked = p.walk->linked;
    info[g] = i;
}

// ---- range decode ---------------------------------------------------------------------------------------------------
// The frames of a range call, as the range kernels read them (device memory): frame f's first byte is at in +
// frame_off[f], its info is info[f] and its entries are index[entry_off[f], + info[f].nblocks).  Range i reads frame
// range_frame[i] (range_frame null: the one-frame call, every range of frame 0).
struct RangeFrames {
    const uint64_t *frame_off;
    const lz4b200_frame_index_info *info;
    const uint64_t *entry_off;
    const uint32_t *range_frame;
};

__device__ __forceinline__ uint32_t frame_of(const RangeFrames &fr, uint32_t i)
{
    return fr.range_frame ? fr.range_frame[i] : 0u;
}

// An info the planners can use, as the one-frame call checks it on the host: a block size the format allows, a block
// count the planner can index, a content length the blocks can hold; and its entries lie in [0, nentries).
__device__ __forceinline__ bool info_ok(const lz4b200_frame_index_info &i, uint64_t entry_off, uint64_t nentries)
{
    const uint64_t bs = i.block_size, nb = i.nblocks;
    const bool bs_ok = bs == (64u << 10) || bs == (256u << 10) || bs == (1u << 20) || bs == (4u << 20) || bs == (8u << 20);
    return nb < 0xffffffffull && (!nb || bs_ok) && i.content_len <= nb * bs && entry_off <= nentries &&
           nb <= nentries - entry_off;
}

// The index comes from outside the library: every info and entry is checked before any is used.  blockIdx.x strides
// over the frames, blockIdx.y over a frame's entries.  Payloads lie inside the frame's region of frame_len[f] bytes and are at most a block; decoded lengths are at
// most a block (a stored block's is its payload); decoded offsets are the running sum of the lengths and end at
// content_len.  sum[0] receives 1 when an info or entry fails.  For the planners, sum[1] and sum[2] receive the largest
// block size among the independent and the linked frames with blocks, and sum[3] bit 0 / bit 1 whether any frame is
// independent / linked.
__global__ void __launch_bounds__(256) index_check_kernel(const RangeFrames fr, const uint64_t *frame_len, uint32_t nf,
                                                          const lz4b200_frame_index_entry *entries, uint64_t nentries,
                                                          uint32_t *sum)
{
    for (uint32_t f = blockIdx.x; f < nf; f += gridDim.x) {
        const lz4b200_frame_index_info i = fr.info[f];
        const uint64_t e0 = fr.entry_off[f];
        const bool lead = blockIdx.y == 0 && threadIdx.x == 0;
        if (!info_ok(i, e0, nentries)) {
            if (lead) atomicOr(sum, 1u);
            continue;
        }
        if (lead) {
            if (i.nblocks) atomicMax(sum + (i.linked ? 2 : 1), (uint32_t)i.block_size);
            atomicOr(sum + 3, i.linked ? 2u : 1u);
        }
        const lz4b200_frame_index_entry *index = entries + e0;
        const uint32_t nb = (uint32_t)i.nblocks;
        const uint64_t n = frame_len[f], bs = i.block_size;
        for (uint32_t b = blockIdx.y * blockDim.x + threadIdx.x; b < nb; b += gridDim.y * blockDim.x) {
            const lz4b200_frame_index_entry e = index[b];
            const uint64_t plen = e.word & 0x7fffffffu;
            const bool stored = (e.word & 0x80000000u) != 0;
            bool ok = e.payload_off <= n && plen <= n - e.payload_off && plen <= bs && e.decoded_len <= bs &&
                      (!stored || e.decoded_len == plen);
            ok = ok && (b == 0 ? e.decoded_off == 0 : e.decoded_off == index[b - 1].decoded_off + index[b - 1].decoded_len);
            if (b == nb - 1) ok = ok && e.decoded_off <= i.content_len && e.decoded_len == i.content_len - e.decoded_off;
            if (!ok) atomicOr(sum, 1u);
        }
    }
}

// Every range's frame is one of the call's nf frames: else sum[0] = 1.
__global__ void __launch_bounds__(128) range_frame_check_kernel(const uint32_t *range_frame, uint32_t nr, uint32_t nf,
                                                                uint32_t *sum)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nr && range_frame[i] >= nf) atomicOr(sum, 1u);
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

// One thread per range of the chunk [r0, r0 + rc) whose frame is independent: its clipped length, its first block (an
// index into the call's entries) and how many blocks it touches.  A linked frame's range touches none here: the linked
// planner serves it.
__global__ void __launch_bounds__(128) range_plan_kernel(const lz4b200_frame_index_entry *index, const RangeFrames fr,
                                                         const uint64_t *start, const uint64_t *len, uint64_t *written,
                                                         uint32_t r0, uint32_t rc, uint32_t *first, uint32_t *count)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rc) return;
    first[i] = 0;
    count[i] = 0;
    const uint32_t f = frame_of(fr, r0 + i);
    const lz4b200_frame_index_info &info = fr.info[f];
    if (info.linked) return;
    uint64_t s, e;
    clip_range(start[r0 + i], len[r0 + i], info.content_len, s, e);
    written[r0 + i] = e - s;
    if (e == s) return;
    const uint32_t e0 = (uint32_t)fr.entry_off[f], nb = (uint32_t)info.nblocks;
    const uint32_t b0 = block_at(index + e0, nb, s), b1 = block_at(index + e0, nb, e - 1);
    first[i] = e0 + b0;
    count[i] = b1 - b0 + 1;
}

// The decode and copy of one (range, block) item of the window [j0, j0 + k), one thread per item (item_off: the
// exclusive scan of the chunk's counts).  A compressed block wholly inside its range decodes into d_out in place, with
// exactly its indexed length as capacity; a partial one into slot j - j0 of the scratch, then its part is copied out; a
// stored block's part is copied from the payload.  Items that decode nothing get in_len 0 and pick 1.  Payload offsets
// are the frame's plus the entry's.
struct RangeItems {
    const lz4b200_frame_index_entry *index;
    RangeFrames fr;
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
    const uint32_t r = lo, f = frame_of(a.fr, a.r0 + r);
    const lz4b200_frame_index_entry e = a.index[a.first[r] + (uint32_t)(j - a.item_off[r])];
    uint64_t s, end;
    clip_range(a.start[a.r0 + r], a.len[a.r0 + r], a.fr.info[f].content_len, s, end);
    const uint64_t d0 = e.decoded_off, d1 = d0 + e.decoded_len;
    const uint64_t from = max(s, d0), to = min(end, d1);
    const bool stored = (e.word & 0x80000000u) != 0, whole = from == d0 && to == d1;
    const uint64_t dst = a.out_off[a.r0 + r] + (from - s), payload = a.fr.frame_off[f] + e.payload_off;
    a.in_off[t] = payload;
    a.in_len[t] = stored ? 0u : (e.word & 0x7fffffffu);
    a.dec_cap[t] = stored ? 0u : e.decoded_len;
    a.want[t] = stored ? 0xffffffffu : e.decoded_len;
    a.dec_off[t] = whole ? dst : a.slot_base + t * a.slot_bytes;
    a.pick[t] = stored ? 1 : 0;
    a.copy_src_a[t] = t * a.slot_bytes + (from - d0);
    a.copy_src_b[t] = payload + (from - d0);
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

// ---- linked frames: marker decode ------------------------------------------------------------------------------------
// A block of a linked frame decodes without the 64 KiB of content before it when every output byte is an entry: the
// byte's value, or a marker naming the earlier entry it copies because its match reaches before the block.  A value
// depends only on compressed bytes, so it is the byte the whole-frame decode gives.  The blocks of a segment (consecutive
// blocks, from a look-back before the blocks the ranges touch) decode in parallel into a window of entries, then markers
// resolve in block order: every marker of a block names one of the 65 535 entries before the block's first, which lie in
// the last 64 KiB of the blocks before it.  Each segment's piece of a window starts with 64 KiB of carry entries: the end
// of the segment's previous piece, or poison for its first.  A byte still poison after resolving copies content before
// the segment, and the segment's look-back is too short.
constexpr uint32_t kMark = 0x80000000u;      // | the window index of the entry a byte copies
constexpr uint32_t kPoison = 0xffffffffu;    // a byte that copies content before its segment
constexpr uint32_t kCarry = 65536;           // carry entries in front of each piece

struct MarkBlock {
    uint64_t payload_off;                    // from d_in[0]: the frame's offset plus the entry's
    uint64_t decoded_off;                    // from the frame's first content byte
    uint32_t word, len;                      // BlockInfo word, indexed decoded length
    uint32_t at;                             // its first entry in the window
};

struct MarkPiece {                           // one segment's blocks in one window
    uint64_t c0, c1;                         // the frame's content [c0, c1)
    uint64_t t0;                             // the segment's first touched byte: its ranges start here or later
    uint32_t blk0, blk1;                     // its blocks in the window's MarkBlock list
    uint32_t base;                           // its carry entries: [base, base + kCarry); its blocks follow
    uint32_t seg;                            // the segment, for the unresolved flag
    uint32_t carried;                        // 1: the carry is the previous window's last piece's end (in carry[])
    uint32_t frame;                          // the segment's frame: a window's pieces ascend by (frame, c0)
};

// One G-lane group per block: the checks of decode_block_linked in the same order, on entries.  Stored blocks are
// values.  A match that reaches before the block's first byte writes markers for that part (its reach before content
// byte 0 is OffsetOutOfBounds, as in the decoder); the rest copies entries with the byte-serial semantics of copy_match,
// so a marker copied inside the block still names an entry before the block.  A block that fails or does not produce
// exactly its indexed length sets *bad.
template <int G>
__global__ void __launch_bounds__(128) marker_decode_kernel(const uint8_t *in, const MarkBlock *blocks, uint32_t nb,
                                                            uint32_t *ent, uint32_t *bad)
{
    const uint32_t lane = threadIdx.x & 31u, sub = lane & (G - 1), leader = lane & ~uint32_t(G - 1);
    const uint32_t gmask = G == 32 ? kFull : (((1u << (G & 31)) - 1u) << leader);
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) / G;
    if (b >= nb) return;
    const MarkBlock bk = blocks[b];
    const uint8_t *__restrict__ src = in + bk.payload_off;
    uint32_t *dst = ent + bk.at;
    const uint32_t n = bk.word & 0x7fffffffu, cap = bk.len;
    if (bk.word & 0x80000000u) {                                   // stored: len == n (checked with the index)
        for (uint32_t i = sub; i < cap; i += G) dst[i] = __ldg(src + i);
        return;
    }
    int32_t status = LZ4B200_OK;
    uint32_t ip = 0, op = 0;
    if (n == 0) status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE;
    while (status == LZ4B200_OK) {
        const uint32_t tok = __ldg(src + ip++);
        uint64_t lit = tok >> 4;
        if (lit == 15) {
            for (;;) {
                if (ip >= n) { status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; break; }
                const uint32_t v = __ldg(src + ip++);
                lit += v;
                if (v != 255) break;
            }
            if (status != LZ4B200_OK) break;
        }
        if (lit) {
            if (lit > (uint64_t)(n - ip)) { status = LZ4B200_DEC_LITERAL_OUT_OF_BOUNDS; break; }
            if (lit > (uint64_t)(cap - op)) { status = LZ4B200_DEC_OUTPUT_TOO_SMALL; break; }
            for (uint32_t i = sub; i < (uint32_t)lit; i += G) dst[op + i] = __ldg(src + ip + i);
            ip += (uint32_t)lit; op += (uint32_t)lit;
        }
        if (ip >= n) break;                                        // the stream ends after literals
        if (n - ip < 2) { status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; break; }
        const uint32_t dist = (uint32_t)__ldg(src + ip) | ((uint32_t)__ldg(src + ip + 1) << 8);
        ip += 2;
        if (dist == 0) { status = LZ4B200_DEC_OFFSET_ZERO; break; }
        uint64_t mlen = 4u + (tok & 15u);
        if (mlen == 19) {
            for (;;) {
                if (ip >= n) { status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; break; }
                const uint32_t v = __ldg(src + ip++);
                mlen += v;
                if (v != 255) break;
            }
            if (status != LZ4B200_OK) break;
        }
        if (dist > op && dist - op > bk.decoded_off) { status = LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS; break; }
        if (mlen > (uint64_t)(cap - op)) { status = LZ4B200_DEC_OUTPUT_TOO_SMALL; break; }
        uint32_t m = (uint32_t)mlen;
        if (dist > op) {                                           // the part before the block: markers
            const uint32_t pre = min(m, dist - op), from = bk.at + op - dist;
            for (uint32_t i = sub; i < pre; i += G) dst[op + i] = kMark | (from + i);
            op += pre; m -= pre;
        }
        __syncwarp(gmask);
        if (m) copy_match<G>(dst + op, dist, m, sub, gmask);
        op += m;
        if (ip >= n) { status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; break; }   // may not end on a match
    }
    if (status != LZ4B200_OK || op != cap) {
        // the block's unwritten entries become poison: the resolve kernels read every entry of the window, and an
        // entry left as whatever the scratch held could pass for a marker naming an entry far outside it
        for (uint32_t i = op + sub; i < cap; i += G) dst[i] = kPoison;
        if (sub == 0) atomicOr(bad, 1u);
    }
}

// Resolve, serial part: one CTA per piece.  The carry is filled first; then, block by block with a barrier between
// them, each block's last min(len, 64 KiB) entries take the entry their marker names, which lies in the carry or in an
// earlier block's last 64 KiB and is already a value or poison.  The other entries are only ever read by the copy-out,
// which resolves them with one more lookup (entries_out_kernel).  Every entry of the window these kernels read has been
// written: the carries here, each block's entries by marker_decode_kernel (poison past the point a failing block
// stopped), so every marker they follow is one the decode wrote.
__global__ void __launch_bounds__(1024) resolve_tails_kernel(const MarkBlock *blocks, const MarkPiece *pieces,
                                                             const uint32_t *carry, uint32_t *ent)
{
    const MarkPiece p = pieces[blockIdx.x];
    uint32_t *c = ent + p.base;
    for (uint32_t i = threadIdx.x; i < kCarry; i += blockDim.x) c[i] = p.carried ? carry[i] : kPoison;
    __syncthreads();
    for (uint32_t b = p.blk0; b < p.blk1; b++) {
        const MarkBlock bk = blocks[b];
        const uint32_t t = min(bk.len, kCarry);
        uint32_t *e = ent + bk.at + (bk.len - t);
        for (uint32_t i = threadIdx.x; i < t; i += blockDim.x) {
            const uint32_t v = e[i];
            if ((v & kMark) && v != kPoison) e[i] = ent[v & ~kMark];
        }
        __syncthreads();
    }
}

// Resolve, parallel part, and copy-out: every range of a linked frame takes its part of the window's pieces of its
// frame (a range lies in one segment, so in at most one piece), one CTA per range at a time.  A marker left (never in a block's last 64 KiB) takes
// the entry it names, which is resolved.  A poison byte is not written; it flags its segment as unresolved.  A range
// that starts before the piece's first touched byte belongs to another segment, whose blocks this one's look-back
// covers: it is skipped, so it neither flags this segment nor is written again.
__global__ void __launch_bounds__(256) entries_out_kernel(const uint32_t *ent, const MarkPiece *pieces, uint32_t np,
                                                          const RangeFrames fr, const uint64_t *start,
                                                          const uint64_t *len, uint8_t *out, const uint64_t *out_off,
                                                          uint32_t nr, uint32_t *unresolved)
{
    for (uint32_t i = blockIdx.x; i < nr; i += gridDim.x) {
        const uint32_t f = frame_of(fr, i);
        if (!fr.info[f].linked) continue;
        uint64_t s, e;
        clip_range(start[i], len[i], fr.info[f].content_len, s, e);
        if (s == e) continue;
        uint32_t lo = 0, hi = np;                                  // the first piece of frame f that ends after s
        while (lo < hi) {
            const uint32_t mid = (lo + hi) / 2;
            if (pieces[mid].frame < f || (pieces[mid].frame == f && pieces[mid].c1 <= s)) lo = mid + 1; else hi = mid;
        }
        for (uint32_t q = lo; q < np && pieces[q].frame == f && pieces[q].c0 < e; q++) {
            const MarkPiece p = pieces[q];
            if (s < p.t0) continue;
            const uint64_t from = max(s, p.c0), to = min(e, p.c1);
            if (from >= to) continue;
            const uint32_t *src = ent + p.base + kCarry + (from - p.c0);
            uint8_t *d = out + out_off[i] + (from - s);
            bool poison = false;
            for (uint64_t x = threadIdx.x; x < to - from; x += blockDim.x) {
                uint32_t v = src[x];
                if ((v & kMark) && v != kPoison) v = ent[v & ~kMark];
                if (v == kPoison) poison = true;
                else d[x] = (uint8_t)v;
            }
            if (poison) unresolved[p.seg] = 1u;
        }
    }
}

// Linked frames: the blocks the ranges touch, as a difference array over the call's entries (touch[first]++,
// touch[last + 1]--), and the clipped length of every range of a linked frame.
__global__ void __launch_bounds__(128) range_touch_kernel(const lz4b200_frame_index_entry *index, const RangeFrames fr,
                                                          const uint64_t *start, const uint64_t *len, uint64_t *written,
                                                          uint32_t nr, int32_t *touch)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nr) return;
    const uint32_t f = frame_of(fr, i);
    const lz4b200_frame_index_info &info = fr.info[f];
    if (!info.linked) return;
    uint64_t s, e;
    clip_range(start[i], len[i], info.content_len, s, e);
    written[i] = e - s;
    if (e == s) return;
    const uint32_t e0 = (uint32_t)fr.entry_off[f], nb = (uint32_t)info.nblocks;
    atomicAdd(touch + e0 + block_at(index + e0, nb, s), 1);
    atomicSub(touch + e0 + block_at(index + e0, nb, e - 1) + 1, 1);
}

}  // namespace fr
}  // namespace lz4b200
