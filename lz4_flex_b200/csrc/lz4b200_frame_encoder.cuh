// lz4b200_frame_encoder.cuh — the host plan of the streaming frame encoder over device memory (lz4b200_frame_encoder).
//
// FrameEncoder (frame/compress.rs:62-404) is an io::Write: write_all, flush and try_finish in any order, any number of
// frames one after another.  The device form keeps one input buffer of whole blocks per encoder.  A call appends its
// input to the buffer; each time the buffer holds a full group of blocks the group is compressed and the buffer empties;
// FLUSH and FINISH compress what is buffered, the last block short, exactly where the reference cuts it.  Only lengths
// decide where blocks are cut and which parse mode (FRESH/CONT) each gets, so the whole call is planned here on the
// host from the encoder's state and the call's length; the device then runs the plan.
// The header also compiles for the host alone (tests/cpp/frame_encoder_host.cpp) for the CPU tests.
#pragma once
#include <stdint.h>

#include <vector>

#include "lz4b200_frame_batch.cuh"

namespace lz4b200 {
namespace fe {

constexpr uint64_t kWindow = 65536;                  // WINDOW_SIZE
constexpr uint64_t kRepositionLimit = 0x7FFFFFFFull; // u32::MAX as usize / 2 (frame/compress.rs:267)

constexpr int kWrite = 0, kFlush = 1, kFinish = 2;   // LZ4B200_ENCODE_WRITE / _FLUSH / _FINISH

static inline uint64_t block_bytes(int id) { return id >= 4 && id <= 7 ? 65536ull << (2 * (id - 4)) : 0; }

// BlockSize::from_buf_length (header.rs:57-67)
static inline int auto_block_id(uint64_t len) { return len > (256u << 10) ? 7 : len > (64u << 10) ? 5 : 4; }

// Blocks per group: as many as fit the frame budget, each taking its input bytes in the buffer and its slot in the
// context's scratch; at least one.
static inline uint64_t group_blocks(uint64_t bs, uint64_t budget)
{
    const uint64_t g = budget / (bs + fb::slot_bytes_for(bs));
    return g ? g : 1;
}

static inline uint32_t header_bytes(const lz4b200_frame_info &info) { return info.has_content_size ? 15u : 7u; }
static inline uint32_t tail_bytes(const lz4b200_frame_info &info) { return info.content_checksum ? 8u : 4u; }
static inline uint32_t block_overhead(const lz4b200_frame_info &info) { return info.block_checksums ? 8u : 4u; }

// What an encoder carries from call to call (the reference's fields of the same names).
struct State {
    int32_t block_size_id = 0;    // frame_info.block_size: 0 (Auto) until the first frame opens, then resolved for good
    uint8_t open = 0;             // is_frame_open
    uint8_t data_written = 0;     // data_to_frame_written: a frame has been finished
    uint64_t group = 0;           // blocks per group of the open (or last) frame, set when it opens
    uint64_t content_len = 0;     // content_len: the frame's input so far, the buffered bytes included
    uint64_t stream_offset = 0;   // src_stream_offset after the last block cut
    uint64_t buffered = 0;        // input bytes in the buffer: whole blocks from its start, the last one partial
};

// One step of a call: copy d_in[src, src + len) to buffer[dst, dst + len) (len may be 0), then, when group_len > 0,
// compress buffer[0, group_len) as nblocks blocks, of which block first_fresh is the first FRESH one (group_plan).
struct Step {
    uint64_t src, dst, len;
    uint64_t group_len;
    uint32_t nblocks, first_fresh;
};

// A call, planned: the header first when the call opens a frame, then the steps, then the EndMark (and the content
// digest) when the call closes the frame cleanly.  status is LZ4B200_FRAME_CONTENT_LENGTH when FINISH finds a content
// length other than the header's: the blocks are written, the frame is closed, no EndMark.
struct CallPlan {
    int status = LZ4B200_OK;
    uint8_t header = 0;
    uint8_t endmark = 0;
    int32_t block_size_id = 0;    // the frame's block size (resolved)
    uint64_t group = 0;           // blocks per group
    std::vector<Step> steps;
    std::vector<uint64_t> block_off;   // src_stream_offset each block is compressed at (after the reposition check)
    State next;
};

// The frame plan of a compressing step: its group's blocks with neither header nor tail.  Only the last block of a
// group can be short, so after the first FRESH block the table repositions every fb::fresh_period blocks.
static inline fb::FramePlan group_plan(const Step &st, uint64_t bs)
{
    fb::FramePlan p{};
    p.in_len = st.group_len;
    p.bs = (uint32_t)bs;
    p.fresh = fb::fresh_period(bs);
    p.first_fresh = st.first_fresh;
    return p;
}

// begin_frame (compress.rs:234-258): resolve Auto from the length of the write that opens the frame, and reset the
// stream state when the frame before had content.  The buffer is empty whenever no frame is open.
static inline void begin_frame(State &s, uint64_t len, uint64_t budget)
{
    s.open = 1;
    if (s.block_size_id == 0) s.block_size_id = auto_block_id(len);
    s.group = group_blocks(block_bytes(s.block_size_id), budget);
    if (s.content_len != 0) {
        s.content_len = 0;
        s.stream_offset = 0;
    }
}

// write_block (compress.rs:261-371) for the blocks of buffer[0, len): each block's parse mode follows the stream offset
// after the reposition check, FRESH exactly when it is 0.  A group without a FRESH block gets first_fresh = nblocks.
static inline void cut_blocks(State &s, CallPlan &p, uint64_t len)
{
    const uint64_t bs = block_bytes(s.block_size_id);
    const uint32_t nblocks = (uint32_t)((len + bs - 1) / bs);
    Step st{0, 0, 0, len, nblocks, nblocks};
    for (uint32_t k = 0; k < nblocks; k++) {
        const uint64_t n = len - k * bs < bs ? len - k * bs : bs;
        if (s.stream_offset + bs + kWindow >= kRepositionLimit) s.stream_offset = 0;   // compress.rs:267-271
        if (s.stream_offset == 0 && st.first_fresh == nblocks) st.first_fresh = k;
        p.block_off.push_back(s.stream_offset);
        s.stream_offset += n;                                                         // compress.rs:366
    }
    s.buffered = 0;
    if (!p.steps.empty() && p.steps.back().group_len == 0) {   // the copy that filled the buffer compresses it
        p.steps.back().group_len = st.group_len;
        p.steps.back().nblocks = st.nblocks;
        p.steps.back().first_fresh = st.first_fresh;
    } else {
        p.steps.push_back(st);
    }
}

// write_all(n bytes), then flush() (op FLUSH) or try_finish() (op FINISH).  `budget` is the context's frame budget,
// which sets the group of a frame the call opens.
static inline CallPlan plan_call(const State &s0, const lz4b200_frame_info &info, uint64_t budget, uint64_t n, int op)
{
    CallPlan p;
    State s = s0;
    if (!s.open && n) {                                       // write (compress.rs:376-378)
        begin_frame(s, n, budget);
        p.header = 1;
    }
    const uint64_t bs = block_bytes(s.block_size_id);
    for (uint64_t pos = 0; pos < n;) {
        const uint64_t cap = s.group * bs;
        const uint64_t take = n - pos < cap - s.buffered ? n - pos : cap - s.buffered;
        p.steps.push_back(Step{pos, s.buffered, take, 0, 0, 0});
        pos += take;
        s.buffered += take;
        s.content_len += take;
        if (s.buffered == cap) cut_blocks(s, p, cap);
    }
    if (op != kWrite && s.buffered) cut_blocks(s, p, s.buffered);   // flush (compress.rs:398-403)
    if (op == kFinish) {                                      // try_finish (compress.rs:173-187)
        if (!s.open && !s.data_written) {
            begin_frame(s, 0, budget);
            p.header = 1;
        }
        s.open = 0;                                           // end_frame (compress.rs:209-230)
        if (info.has_content_size && info.content_size != s.content_len) {
            p.status = LZ4B200_FRAME_CONTENT_LENGTH;
        } else {
            p.endmark = 1;
            s.data_written = 1;
        }
    }
    p.block_size_id = s.block_size_id;
    p.group = s.group;
    p.next = s;
    return p;
}

// The most bytes plan_call(s, info, budget, n, op) writes: the header when the call opens a frame, 4 + length (+ 4 with
// block checksums) for every block of every group the call completes (a block that does not shrink is stored), and the
// EndMark (+ digest) for FINISH.
static inline uint64_t call_bound(const State &s, const lz4b200_frame_info &info, uint64_t budget, uint64_t n, int op)
{
    uint64_t b = 0, buffered = s.buffered, group = s.group;
    int id = s.block_size_id;
    bool open = s.open != 0;
    if (!open && n) {
        b += header_bytes(info);
        if (!id) id = auto_block_id(n);
        group = group_blocks(block_bytes(id), budget);
        open = true;
    }
    const uint64_t bs = block_bytes(id), total = buffered + n;
    uint64_t done = 0, nb = 0;
    if (total) {
        if (op == kWrite) {
            done = total / (group * bs) * (group * bs);
            nb = done / bs;
        } else {
            done = total;
            nb = (total + bs - 1) / bs;
        }
    }
    b += done + nb * block_overhead(info);
    if (op == kFinish) {
        if (!open && !s.data_written) b += header_bytes(info);
        b += tail_bytes(info);
    }
    return b;
}

}  // namespace fe
}  // namespace lz4b200
