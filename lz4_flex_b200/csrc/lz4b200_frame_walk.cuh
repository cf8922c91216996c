// lz4b200_frame_walk.cuh — the LZ4 frame container walk and XXH32, shared by the host and the device.
//
// A frame is a header, a chain of BlockInfo words each followed by its payload (and a block checksum when the header
// asks for one), an EndMark and an optional content checksum (src/frame/header.rs, src/frame/decompress.rs:109-342).
// frame_walk() parses the header and follows the chain, recording one FrameBlockDesc (16 bytes) per block; it never
// reads a byte at or past `n`.  The same code runs on the CPU for frames in host memory (lz4b200_frame_decompress_next)
// and in one GPU thread for frames in device memory (lz4b200_frame_decompress_next_device), so both calls see the same
// blocks and stop with the same status at the same byte.  Words are assembled from bytes: the input may have any
// alignment.  Block checksums are recorded, not checked: verifying them is a separate step (block_checksum_ok, one
// thread per block on the GPU), and frame_walk_fail_block() cuts the walk at the first block that fails.
// The header also compiles for the host alone (tests/cpp/frame_walk_host.cpp) for the CPU tests.
#pragma once
#include <stdint.h>

#include "../../include/lz4b200.h"

#if defined(__CUDACC__)
#define FW_FN __host__ __device__ __forceinline__
#else
#define FW_FN static inline
#endif

namespace lz4b200 {
namespace fw {

// ---- XXH32 (twox-hash XxHash32): header, block and content checksums --------------------------------------------------
constexpr uint32_t kP1 = 2654435761u, kP2 = 2246822519u, kP3 = 3266489917u, kP4 = 668265263u, kP5 = 374761393u;

FW_FN uint32_t rd32(const uint8_t *p)
{
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}
FW_FN uint32_t rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
FW_FN uint32_t xxh32_round(uint32_t a, uint32_t v) { return rotl(a + v * kP2, 13) * kP1; }

FW_FN void xxh32_reset(lz4b200_xxh32_state &st, uint32_t seed)
{
    st.acc[0] = seed + kP1 + kP2; st.acc[1] = seed + kP2; st.acc[2] = seed; st.acc[3] = seed - kP1;
    for (int i = 0; i < 16; i++) st.buf[i] = 0;
    st.fill = 0; st.seed = seed; st.total = 0;
}

FW_FN void xxh32_stripe(uint32_t acc[4], const uint8_t *p)
{
    for (int i = 0; i < 4; i++) acc[i] = xxh32_round(acc[i], rd32(p + 4 * i));
}

FW_FN void xxh32_update(lz4b200_xxh32_state &st, const uint8_t *p, uint64_t n)
{
    st.total += n;
    if (st.fill) {
        while (n && st.fill < 16) { st.buf[st.fill++] = *p++; n--; }
        if (st.fill < 16) return;
        xxh32_stripe(st.acc, st.buf);
        st.fill = 0;
    }
    uint32_t acc[4] = {st.acc[0], st.acc[1], st.acc[2], st.acc[3]};
    for (; n >= 16; p += 16, n -= 16) xxh32_stripe(acc, p);
    for (int i = 0; i < 4; i++) st.acc[i] = acc[i];
    for (uint32_t i = 0; i < (uint32_t)n; i++) st.buf[i] = p[i];
    st.fill = (uint32_t)n;
}

FW_FN uint32_t xxh32_digest(const lz4b200_xxh32_state &st)
{
    uint32_t h = st.total >= 16 ? rotl(st.acc[0], 1) + rotl(st.acc[1], 7) + rotl(st.acc[2], 12) + rotl(st.acc[3], 18)
                                : st.seed + kP5;
    h += (uint32_t)st.total;
    const uint8_t *p = st.buf, *e = st.buf + st.fill;
    for (; p + 4 <= e; p += 4) h = rotl(h + rd32(p) * kP3, 17) * kP4;
    for (; p < e; p++) h = rotl(h + (*p) * kP5, 11) * kP1;
    h ^= h >> 15; h *= kP2; h ^= h >> 13; h *= kP3; h ^= h >> 16;
    return h;
}

FW_FN uint32_t xxh32(const uint8_t *p, uint64_t n, uint32_t seed)
{
    lz4b200_xxh32_state st;
    xxh32_reset(st, seed);
    xxh32_update(st, p, n);
    return xxh32_digest(st);
}

// ---- the walk ---------------------------------------------------------------------------------------------------------
struct FrameBlockDesc {            // one block of a frame, 16 bytes
    uint64_t payload_off;          // from the start of the frame
    uint32_t word;                 // the BlockInfo word: payload length | 0x80000000 for a stored (uncompressed) block
    uint32_t checksum;             // the stored block checksum (0 when the frame has none)
};
FW_FN uint32_t block_len(const FrameBlockDesc &b) { return b.word & 0x7fffffffu; }
FW_FN bool block_stored(const FrameBlockDesc &b) { return (b.word & 0x80000000u) != 0; }

enum : uint32_t { kWalkHeader = 0, kWalkBlocks = 1, kWalkDone = 2 };
constexpr uint32_t kNoBlock = 0xffffffffu;

struct FrameWalk {
    uint64_t ip = 0;               // next byte to read; once done: the bytes the frame consumed
    uint64_t bs = 0;               // the frame's maximum block size
    uint64_t content_size = 0;
    uint64_t nblocks = 0;          // blocks recorded so far
    int32_t status = LZ4B200_OK;   // what stopped the walk: a header error, BlockTooBig, EOF (or, after the verify step,
                                   // the block checksum)
    uint32_t stage = kWalkHeader;
    uint32_t flg = 0x20;           // the FLG byte (legacy frames: independent blocks, no checksums)
    uint32_t content_checksum = 0;
    uint8_t has_size = 0, has_checksum = 0, closed = 0, linked = 0;
    uint32_t pad = 0;
};

FW_FN uint64_t block_size_bytes(int id) { return id >= 4 && id <= 7 ? (64ull << 10) << (2 * (id - 4)) : 0; }

// read_frame_info — frame/decompress.rs:109-176, frame/header.rs:277-355.  Header errors consume nothing; input that
// ends inside the header consumes all of it.
FW_FN void walk_header(const uint8_t *in, uint64_t n, FrameWalk &w)
{
    w.stage = kWalkDone;
    if (n == 0) return;                                         // 0 bytes where a frame would start: end of data
    if (n < 4) { w.ip = n; w.status = LZ4B200_FRAME_IO_EOF; return; }
    const uint32_t magic = rd32(in);
    if (magic == 0x184C2102u) {                                 // legacy frame: header.rs:285-291
        w.ip = 4; w.bs = 8u << 20; w.flg = 0x20; w.stage = kWalkBlocks;
        return;
    }
    if (n == 4) { w.ip = 4; return; }                           // decompress.rs:124-128: nothing after the magic
    if (n < 7) { w.ip = n; w.status = LZ4B200_FRAME_IO_EOF; return; }
    if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) { w.status = LZ4B200_FRAME_SKIPPABLE; return; }
    if (magic != 0x184D2204u) { w.status = LZ4B200_FRAME_WRONG_MAGIC; return; }
    const uint32_t flg = in[4], bd = in[5];
    const uint64_t need = 7 + ((flg & 0x08) ? 8 : 0) + ((flg & 0x01) ? 4 : 0);
    if (n < need) { w.ip = n; w.status = LZ4B200_FRAME_IO_EOF; return; }
    if ((flg & 0xC0) != 0x40) { w.status = LZ4B200_FRAME_UNSUPPORTED_VERSION; return; }
    if ((flg & 0x02) || (bd & 0x8F)) { w.status = LZ4B200_FRAME_RESERVED_BITS; return; }
    const int id = (bd >> 4) & 7;
    if (id < 4) { w.status = LZ4B200_FRAME_UNSUPPORTED_BLOCKSIZE; return; }
    uint64_t o = 6;
    if (flg & 0x08) {
        w.content_size = (uint64_t)rd32(in + o) | ((uint64_t)rd32(in + o + 4) << 32);
        w.has_size = 1;
        o += 8;
    }
    if (flg & 0x01) o += 4;
    if ((uint8_t)(xxh32(in + 4, o - 4, 0) >> 8) != in[o]) { w.status = LZ4B200_FRAME_HEADER_CHECKSUM; return; }
    if (flg & 0x01) { w.status = LZ4B200_FRAME_DICTIONARY; return; }
    w.flg = flg;
    w.bs = block_size_bytes(id);
    w.linked = !(flg & 0x20);
    w.ip = o + 1;
    w.stage = kWalkBlocks;
}

// Parses the header on the first call, then follows the BlockInfo chain (decompress.rs:189-342) and records at most
// `max_blocks` blocks into `out`; call again with the same `w` until w.stage == kWalkDone.  Returns the blocks recorded.
FW_FN uint32_t frame_walk(const uint8_t *in, uint64_t n, FrameWalk &w, FrameBlockDesc *out, uint32_t max_blocks)
{
    if (w.stage == kWalkHeader) walk_header(in, n, w);
    uint32_t k = 0;
    uint64_t ip = w.ip;
    while (w.stage == kWalkBlocks && k < max_blocks) {
        if (n - ip < 4) { ip = n; w.stage = kWalkDone; break; }    // EOF where a BlockInfo is due: decompress.rs:236-243
        const uint32_t word = rd32(in + ip);
        ip += 4;
        if (word == 0) {                                            // EndMark
            w.closed = 1;
            w.stage = kWalkDone;
            if (w.flg & 0x04) {
                if (n - ip < 4) { w.status = LZ4B200_FRAME_IO_EOF; ip = n; break; }
                w.has_checksum = 1;
                w.content_checksum = rd32(in + ip);
                ip += 4;
            }
            break;
        }
        const uint64_t len = word & 0x7fffffffu;
        if (len > w.bs) { w.status = LZ4B200_FRAME_BLOCK_TOO_BIG; w.stage = kWalkDone; break; }
        if (n - ip < len) { w.status = LZ4B200_FRAME_IO_EOF; ip = n; w.stage = kWalkDone; break; }
        const uint64_t payload = ip;
        ip += len;
        uint32_t checksum = 0;
        if (w.flg & 0x10) {
            if (n - ip < 4) { w.status = LZ4B200_FRAME_IO_EOF; ip = n; w.stage = kWalkDone; break; }
            checksum = rd32(in + ip);
            ip += 4;
        }
        out[k++] = FrameBlockDesc{payload, word, checksum};
    }
    w.ip = ip;
    w.nblocks += k;
    return k;
}

// ---- the walk over a frame that arrives in chunks (lz4b200_frame_decoder) ---------------------------------------------
// Bytes the unit at p[0, avail) takes: the header, a block (BlockInfo, payload, block checksum) or the EndMark with the
// content checksum.  While p[] is too short to tell, the bytes that tell more (4, then 7 for a header); a unit the walk
// rejects from its first bytes (a bad magic, BlockTooBig) takes no more than those.
FW_FN uint64_t walk_unit_bytes(const uint8_t *p, uint64_t avail, const FrameWalk &w)
{
    if (avail < 4) return 4;
    if (w.stage == kWalkHeader) {
        const uint32_t magic = rd32(p);
        if (magic == 0x184C2102u) return 4;
        if (avail < 7 || magic != 0x184D2204u) return 7;
        return 7 + ((p[4] & 0x08) ? 8 : 0) + ((p[4] & 0x01) ? 4 : 0);
    }
    const uint32_t word = rd32(p);
    if (word == 0) return 4 + ((w.flg & 0x04) ? 4 : 0);
    const uint64_t len = word & 0x7fffffffu;
    if (len > w.bs) return 4;
    return 4 + len + ((w.flg & 0x10) ? 4 : 0);
}

// frame_walk over a frame presented in chunks.  in[0, n) holds the frame's bytes from w.ip on: a call starts where the
// last one stopped, and w.ip stays an offset from the frame's first byte.  Recorded payload offsets are from in[0].  It
// takes whole units only, at most max_blocks blocks.  Unless `eof` (in[0, n) runs to the end of the input), it stops
// before a unit in[] does not hold whole, with no status set, and *need receives the bytes from that unit's start it
// needs at least; otherwise *need = 0.  With `eof` a truncated unit ends the walk as frame_walk ends it.  So any
// chunking of a frame, `eof` on the last chunk, records the blocks frame_walk records and leaves the same FrameWalk.
// It never reads at or past n.
FW_FN uint32_t frame_walk_stream(const uint8_t *in, uint64_t n, bool eof, FrameWalk &w, FrameBlockDesc *out,
                                 uint32_t max_blocks, uint64_t *need)
{
    const uint64_t at = w.ip;
    uint32_t k = 0;
    *need = 0;
    while (w.stage != kWalkDone && k < max_blocks) {
        const uint64_t rel = w.ip - at;
        const uint64_t unit = walk_unit_bytes(in + rel, n - rel, w);
        if (!eof && unit > n - rel) { *need = unit; break; }
        const uint64_t lim = eof ? n : rel + unit;
        if (w.stage == kWalkHeader) { walk_header(in, lim, w); continue; }   // only ever at the frame's first byte
        FrameWalk u = w;
        u.ip = rel;
        k += frame_walk(in, lim, u, out + k, 1);
        u.ip += at;
        w = u;
    }
    return k;
}

// The block checksum (frame/decompress.rs:258-266): XXH32 of the payload as stored.
FW_FN bool block_checksum_ok(const uint8_t *in, const FrameBlockDesc &b)
{
    return xxh32(in + b.payload_off, block_len(b), 0) == b.checksum;
}

// The frame as the reader leaves it when block k (recorded by the walk) fails its checksum: blocks [0, k) are
// delivered, the input is consumed up to the end of block k's payload, and the error is BlockChecksumError.
FW_FN void frame_walk_fail_block(FrameWalk &w, const FrameBlockDesc &b, uint32_t k)
{
    w.nblocks = k;
    w.status = LZ4B200_FRAME_BLOCK_CHECKSUM;
    w.ip = b.payload_off + block_len(b);
    w.closed = 0;
    w.has_checksum = 0;
}

// ---- group planning, shared by the one-frame group loop and the batch decoder -------------------------------------------
// Upper bound of what one block can decode to: its frame's block size, and never more than 255 output bytes per
// input byte (a length-extension byte of 0xFF stands for 255 bytes; nothing in the format is denser).
FW_FN uint64_t block_decoded_cap(uint64_t payload_len, uint64_t bs)
{
    const uint64_t c = payload_len * 255ull + 16ull;
    return bs < c ? bs : c;
}
// The device slot a block decodes into: its cap rounded up to 16 bytes (stored blocks are only gathered: none).
FW_FN uint64_t block_slot_cap(const FrameBlockDesc &b, uint64_t bs) { return block_stored(b) ? 0 : block_decoded_cap(block_len(b), bs); }
FW_FN uint64_t slot_bytes(uint64_t cap) { return (cap + 15) & ~15ull; }

// The group loop's cut: a group that already holds blocks whose slots take `slot_total` bytes ends before a block
// whose slot needs `cap` bytes, or whose payload ends `in_span` bytes past the group's first payload, when either would
// pass the budget.
FW_FN bool group_cut(uint64_t slot_total, uint64_t cap, uint64_t in_span, uint64_t budget)
{
    return slot_total + cap > budget || in_span > budget;
}

// What the batch decoder plans with for one frame (32 bytes): its blocks, their slot bytes, whether it is decoded as
// one linked chain, and whether the group loop would decode it as one group (linked frames always are).
struct FrameCount {
    uint64_t slot_total = 0;
    uint64_t nblocks = 0;
    uint64_t first_off = 0;        // payload offset of block 0
    uint8_t linked = 0, one_group = 1;
};

// Adds the next block (stream order) of a frame to its count.
FW_FN void frame_count_add(FrameCount &c, const FrameBlockDesc &b, uint64_t bs, uint64_t budget)
{
    const uint64_t cap = block_slot_cap(b, bs);
    if (c.nblocks == 0) c.first_off = b.payload_off;
    else if (group_cut(c.slot_total, cap, b.payload_off + block_len(b) - c.first_off, budget)) c.one_group = 0;
    c.slot_total += slot_bytes(cap);
    c.nblocks++;
}

// The whole walk of the frame at in[0, n) with a small descriptor buffer, keeping only the count; w is left as the walk
// ends (before any block checksum is checked).
FW_FN void frame_count(const uint8_t *in, uint64_t n, FrameWalk &w, FrameCount &c, uint64_t budget)
{
    FrameBlockDesc buf[4];
    c = FrameCount{};
    while (w.stage != kWalkDone) {
        const uint32_t k = frame_walk(in, n, w, buf, 4);
        for (uint32_t i = 0; i < k; i++) frame_count_add(c, buf[i], w.bs, budget);
    }
    if (w.linked) c.one_group = 1;                  // one dependency chain: the group loop never cuts it
    c.linked = w.linked && c.nblocks > 1;
}

}  // namespace fw

// ---- the frame decoders' group pipeline ---------------------------------------------------------------------------------
// Every frame decoder decodes a frame group by group through the same kernels: arguments, decode, resolve, gather,
// content hash, digest (decode_group in lz4b200_api.cu).  A group holds the blocks of one or more frames, described by
// one GroupFrame each: the batch decoder's record walk fills one per frame, the group loop (decode_frame_blocks) one per
// group of a frame.  Blocks are indexed frame after frame, the blocks of independent frames first and those of linked
// frames after them.  The frame index (lz4b200_frame_range.cuh) sizes the blocks of such groups and runs their result
// step.
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

}  // namespace lz4b200
