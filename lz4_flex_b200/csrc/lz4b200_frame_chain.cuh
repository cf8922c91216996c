// lz4b200_frame_chain.cuh — the per-block plan of a BlockMode::Linked frame, shared by the host and the device.
//
// In a linked frame every block may match into the 64 KiB before it, and lz4_flex's FrameEncoder carries one hash table
// from block to block (frame/compress.rs:261-371).  What a block's parse can reach is decided by the encoder's buffer
// moves (:327-356), which depend only on the block lengths, and by the table reposition of :266-271.  chain_next runs
// that state machine one block at a time and gives, for each block:
//   - stream:   S, the table coordinate of the compressor's input slice's first byte (input_stream_offset);
//   - ext_len:  E, the ext_dict length: the stream bytes [S - E, S), which are the E frame bytes before the slice;
//   - prefix:   input_pos, the bytes of the slice before the block (the frame bytes right before it);
//   - shift:    when `reposition`, every table entry drops by shift, saturating at 0, before the block;
//   - to_frame: frame position = table coordinate + to_frame;
//   - first:    position 0 goes into the table before the parse (compress.rs:353-359: input_pos == 0 && S == 0).
// A candidate at or after S extends like any in-input match and backwards to the slice's first byte; an ext_dict
// candidate stops at S going forwards (count_same_bytes, compress.rs:156-170) and at S - E going backwards.
// The input is block lengths, not a block size, so that an encoder with flushes (short blocks) runs the same plan.
// The header also compiles for the host alone (tests/cpp/frame_chain_host.cpp) for the CPU tests.
#pragma once
#include "lz4b200_frame_walk.cuh"

namespace lz4b200 {
namespace fb {

constexpr uint64_t kChainWindow = 65536;             // WINDOW_SIZE

// The encoder's buffer state between blocks.
struct ChainState {
    uint64_t src_start;      // bytes of the buffer before the next block (its prefix)
    uint64_t ext_len;        // ext_dict length
    uint64_t stream;         // src_stream_offset
    uint64_t consumed;       // frame bytes before the next block
    uint64_t bs;             // the frame's block size
};

struct ChainBlock {
    uint64_t stream;
    uint64_t shift;
    int64_t to_frame;
    uint32_t ext_len;
    uint32_t prefix;
    bool reposition;
    bool first;
};

// A frame opens with an empty buffer, no ext_dict and stream offset 0 (begin_frame, frame/compress.rs:244-255).
FW_FN ChainState chain_start(uint64_t bs)
{
    ChainState c;
    c.src_start = 0; c.ext_len = 0; c.stream = 0; c.consumed = 0; c.bs = bs;
    return c;
}

// The plan of the next block, of `len` bytes (1 <= len <= bs), and the state after it.
FW_FN ChainBlock chain_next(ChainState &c, uint64_t len)
{
    ChainBlock b;
    b.reposition = c.stream + c.bs + kChainWindow >= 0x7FFFFFFFull;        // :266-271, u32::MAX / 2
    b.shift = 0;
    if (b.reposition) {
        b.shift = c.stream - c.ext_len;
        c.stream = c.ext_len;
    }
    b.stream = c.stream;
    b.ext_len = (uint32_t)c.ext_len;
    b.prefix = (uint32_t)c.src_start;
    b.to_frame = (int64_t)(c.consumed - c.src_start) - (int64_t)c.stream;
    b.first = c.src_start == 0 && c.stream == 0;
    // buffer moves after the block (:324-356)
    c.consumed += len;
    c.src_start += len;
    if (c.src_start >= c.bs + kChainWindow) {       // the last 64 KiB become the ext_dict, input restarts at the buffer's head
        c.ext_len = kChainWindow;
        c.stream += c.src_start;
        c.src_start = 0;
    } else if (c.src_start + c.ext_len > kChainWindow) {   // prefix and ext_dict hold more than 64 KiB: shrink the ext_dict
        const uint64_t over = c.src_start + c.ext_len - kChainWindow;
        c.ext_len -= over < c.ext_len ? over : c.ext_len;
    }
    return b;
}

}  // namespace fb
}  // namespace lz4b200
