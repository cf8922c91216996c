// lz4b200_frame_batch.cuh — the plan every frame encoder runs (lz4b200_frame_compress, _compress_device,
// _compress_batch_device and the streaming encoder's groups), shared by the host and the device.
//
// The host plans every frame of a batch in one pass (plan_frame) and hands the table to the device.  The blocks of all
// frames are numbered frame after frame and compressed in one launch; one GPU thread per block finds its frame by
// binary search over the frames' first block indices and derives its input range, its scratch slot, its parse mode and
// where its [BlockInfo | payload (| checksum)] segment lands in the packed output (batch_block).  Frames lie back to
// back: frame f starts at seg_off[first_block] + ovh, where seg_off is the exclusive scan of every block's segment size
// and ovh the header, EndMark and digest bytes of the frames before it (frame_place).
// The sync-free batch call plans its frames on the device instead (batch_frame, capacity_status, frame_extent and
// place_frame in one CTA's scan), from the same functions.
// The header also compiles for the host alone (tests/cpp/frame_batch_host.cpp, frame_batch_async_host.cpp) for the CPU
// tests.
#pragma once
#include "lz4b200_frame_walk.cuh"

namespace lz4b200 {
namespace fb {

// One frame of the batch, 64 bytes.
struct FramePlan {
    uint64_t in_off, in_len;       // the frame's input: d_in[in_off, in_off + in_len)
    uint64_t slot_base;            // scratch bytes of the blocks of the frames before
    uint64_t ovh;                  // header, EndMark and digest bytes of the frames before
    uint32_t first_block;          // batch index of the frame's block 0
    uint32_t bs;                   // the frame's block size
    uint32_t fresh;                // table epoch (frame/compress.rs:266-271): block k of the frame is FRESH iff
                                   // k >= first_fresh and (k - first_fresh) % fresh == 0
    uint8_t hdr[15];               // FrameInfo::write (header.rs:232-275): at most 15 bytes without a dictionary id
    uint8_t hdr_len;
    uint32_t first_fresh;          // 0 for a whole frame; after a flush a streaming group's epochs are off its block grid
};

// The scratch slot of a block of `len` input bytes: lz4b200_max_output_size(len) rounded up to 16 bytes.
FW_FN uint64_t slot_bytes_for(uint64_t len) { return (20ull + len * 110ull / 100ull + 15ull) & ~15ull; }

// Full blocks of bs bytes that share one table epoch: FrameEncoder repositions its table at the first block whose
// stream offset off has off + bs + 64 KiB >= 2^31 - 1 (frame/compress.rs:266-271).
FW_FN uint32_t fresh_period(uint64_t bs)
{
    const uint64_t limit = 0x7FFFFFFFull - 65536ull - bs;
    return (uint32_t)((limit + bs - 1) / bs);
}

FW_FN uint64_t frame_blocks(const FramePlan &p) { return (p.in_len + p.bs - 1) / p.bs; }

// Scratch of a frame: a slot per full block, and one sized for the last block's length.
FW_FN uint64_t frame_slot_bytes(const FramePlan &p)
{
    const uint64_t nb = frame_blocks(p);
    return nb ? (nb - 1) * slot_bytes_for(p.bs) + slot_bytes_for(p.in_len - (nb - 1) * p.bs) : 0;
}

// Completes p, whose input, block size, table period and header are set, from the frame before it (null: p is the
// first).  `tail_len` is the EndMark and digest bytes every frame of the batch ends with (4, or 8 with a content
// checksum).  The caller checks that the batch's blocks fit first_block.
FW_FN void plan_frame(FramePlan &p, const FramePlan *prev, uint32_t tail_len)
{
    p.first_block = prev ? prev->first_block + (uint32_t)frame_blocks(*prev) : 0u;
    p.slot_base = prev ? prev->slot_base + frame_slot_bytes(*prev) : 0u;
    p.ovh = prev ? prev->ovh + prev->hdr_len + tail_len : 0u;
}

// The frame that holds batch block b: the last frame whose first block is at or before b (frames without blocks share
// their successor's first block and come before it).
FW_FN uint32_t find_frame(const FramePlan *p, uint32_t nframes, uint32_t b)
{
    uint32_t lo = 0, hi = nframes;                   // p[lo].first_block <= b, and b < p[hi].first_block or hi == nframes
    while (hi - lo > 1) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (p[mid].first_block <= b) lo = mid;
        else hi = mid;
    }
    return lo;
}

// What the compressor, the pack and the block checksums need of batch block b.
struct BlockJob {
    uint64_t in_off;               // input at d_in + in_off
    uint64_t out_off;              // scratch slot
    uint64_t dst_shift;            // the packed segment lands at seg_off[b] + dst_shift
    uint32_t in_len, out_cap;
    uint32_t frame, k;             // frame and frame-local index
    uint8_t flags;                 // LZ4B200_BLOCK_* parse mode
};

FW_FN BlockJob batch_block(const FramePlan *p, uint32_t nframes, uint32_t b)
{
    BlockJob j;
    j.frame = find_frame(p, nframes, b);
    const FramePlan &q = p[j.frame];
    j.k = b - q.first_block;
    const uint64_t o = (uint64_t)j.k * q.bs, rem = q.in_len - o;
    j.in_off = q.in_off + o;
    j.in_len = (uint32_t)(rem < q.bs ? rem : q.bs);
    j.out_off = q.slot_base + (uint64_t)j.k * slot_bytes_for(q.bs);
    j.out_cap = (uint32_t)slot_bytes_for(j.in_len);
    j.dst_shift = q.ovh + q.hdr_len;
    const bool fresh = j.k >= q.first_fresh && (j.k - q.first_fresh) % q.fresh == 0;
    j.flags = (uint8_t)(LZ4B200_BLOCK_HASH5_ALWAYS | (fresh ? 0u : LZ4B200_BLOCK_CONT));
    return j;
}

// Where frame p lies in the packed output, given the scan of the segment sizes: its header at *start, its EndMark at
// *endmark (the digest, when there is one, follows it).
FW_FN void frame_place(const FramePlan &p, const uint64_t *seg_off, uint64_t *start, uint64_t *endmark)
{
    *start = seg_off[p.first_block] + p.ovh;
    *endmark = seg_off[p.first_block + frame_blocks(p)] + p.ovh + p.hdr_len;
}

// ---- the header, shared by the host entry points and the device planner ------------------------------------------------

// BlockSize::from_buf_length — frame/header.rs:57-67
FW_FN int auto_block_size_id(uint64_t first_write_len)
{
    if (first_write_len > (256u << 10)) return 7;
    if (first_write_len > (64u << 10)) return 5;
    return 4;
}

// FrameInfo::write — frame/header.rs:232-275: the header's bytes at out, their count (at most 15), or 0 when cap cannot
// hold them.
FW_FN uint32_t write_header(const lz4b200_frame_info &info, uint8_t *out, uint64_t cap)
{
    uint8_t buf[15] = {0x04, 0x22, 0x4D, 0x18};
    uint32_t o = 4;
    uint8_t flg = 0x40;
    if (info.block_checksums) flg |= 0x10;
    if (info.content_checksum) flg |= 0x04;
    if (!info.linked) flg |= 0x20;
    if (info.has_content_size) flg |= 0x08;
    buf[o++] = flg;
    buf[o++] = (uint8_t)(info.block_size_id << 4);
    if (info.has_content_size)
        for (int i = 0; i < 8; i++) buf[o++] = (uint8_t)(info.content_size >> (8 * i));
    buf[o] = (uint8_t)(fw::xxh32(buf + 4, o - 4, 0) >> 8);
    o++;
    if (cap < o) return 0;
    for (uint32_t i = 0; i < o; i++) out[i] = buf[i];
    return o;
}

// lz4b200_frame_bound for n input bytes in blocks of bs: the header at its longest, every block's BlockInfo and
// checksum, the EndMark and the digest.
FW_FN uint64_t frame_bound_bytes(uint64_t n, uint64_t bs) { return 19 + n + (n + bs - 1) / bs * 8 + 8; }

// Sets what `info` (block size resolved) and the input d_in[in_off, in_off + in_len) decide of the zeroed plan p, the
// header included; plan_frame places it after the frame before.  p is filled in place, not returned: copying a
// returned plan into the batch's table stalls the host on every frame.
FW_FN void frame_plan(FramePlan &p, const lz4b200_frame_info &info, uint64_t in_off, uint64_t in_len)
{
    p.in_off = in_off;
    p.in_len = in_len;
    p.bs = (uint32_t)fw::block_size_bytes(info.block_size_id);
    p.fresh = fresh_period(p.bs);
    p.hdr_len = (uint8_t)write_header(info, p.hdr, sizeof p.hdr);
}

// ---- the sync-free batch planner (lz4b200_frame_compress_batch_device_async) -------------------------------------------
// One CTA scans the frames on the device.  Frame f is planned only if frames 0..f together fit the three limits; since
// every frame adds a non-negative amount to each sum, the frames inside form a prefix.  A frame past them keeps its
// place but has no input and no header (in_len = 0, hdr_len = 0): no blocks, and nothing of it is written.

// Saturating: a sum that would wrap stays past every limit.
FW_FN uint64_t sat_add(uint64_t a, uint64_t b) { return a + b < a ? ~0ull : a + b; }

struct BatchLimits {
    uint64_t blocks, in_bytes, out_bytes;   // max_blocks, max_in_bytes, out_cap
};

// What one frame adds to the sums the capacity rule checks.
struct FrameCost {
    uint64_t blocks, in_bytes, bound;       // blocks, input bytes, lz4b200_frame_bound bytes
};

// Frame f of the batch, before placement: its plan under *info (Auto resolved from in_len, the content size in_len) and
// its cost.  A frame of 2^62 bytes or more has more than 2^32 blocks, past every capacity: its cost is taken at 2^62
// bytes, so that no sum wraps.
FW_FN FrameCost batch_frame(FramePlan &p, const lz4b200_frame_info &info, uint64_t in_off, uint64_t in_len)
{
    lz4b200_frame_info fi = info;
    if (fi.block_size_id == 0) fi.block_size_id = auto_block_size_id(in_len);                  // compress.rs:236-238
    fi.content_size = in_len;
    frame_plan(p, fi, in_off, in_len);
    const uint64_t n = in_len < (1ull << 62) ? in_len : (1ull << 62);
    FrameCost c;
    c.blocks = (n + p.bs - 1) / p.bs;
    c.in_bytes = n;
    c.bound = frame_bound_bytes(n, p.bs);
    return c;
}

// The status of a frame whose frames 0..f sum to `incl`: OK inside all three limits; else the first limit passed, in
// the order blocks, input bytes, bound, decides: INVALID_ARGUMENT for the first two, COMPRESS_OUTPUT_TOO_SMALL for the
// bound.
FW_FN int32_t capacity_status(const FrameCost &incl, const BatchLimits &lim)
{
    if (incl.blocks > lim.blocks || incl.in_bytes > lim.in_bytes) return LZ4B200_INVALID_ARGUMENT;
    if (incl.bound > lim.out_bytes) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    return LZ4B200_OK;
}

// A frame past capacity: no blocks, no header.
FW_FN void drop_frame(FramePlan &p) { p.in_len = 0; p.hdr_len = 0; }

// What frame p adds to the places of the frames after it (plan_frame's sums): its blocks, its scratch and its header,
// EndMark and digest bytes.  A dropped frame adds nothing.
struct FramePlace {
    uint64_t blocks, slot, ovh;
};
FW_FN FramePlace frame_extent(const FramePlan &p, uint32_t tail_len)
{
    FramePlace e;
    e.blocks = frame_blocks(p);
    e.slot = frame_slot_bytes(p);
    e.ovh = p.hdr_len ? p.hdr_len + tail_len : 0u;
    return e;
}

// Places p after frames whose extents sum to `before`.
FW_FN void place_frame(FramePlan &p, const FramePlace &before)
{
    p.first_block = (uint32_t)before.blocks;
    p.slot_base = before.slot;
    p.ovh = before.ovh;
}

}  // namespace fb
}  // namespace lz4b200
