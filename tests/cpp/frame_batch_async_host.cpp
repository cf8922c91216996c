// Host build of the sync-free batch frame encoder's planner (lz4_flex_b200/csrc/lz4b200_frame_batch.cuh): the per-frame
// plan, cost, capacity status, drop and placement that frame_async_plan_kernel runs in one CTA's scan, here run frame
// after frame, and the shared header writer.  Compiled by g++ with AddressSanitizer and UndefinedBehaviorSanitizer and
// driven by tests/test_frame_batch_async_host.py.  Test infrastructure only: nothing in the product links or runs this.
//
// stdin: records, each a u32 kind:
//   0 (batch):  i32 block_size_id | i32 block_checksums | i32 content_checksum | i32 has_content_size | i32 linked |
//               u64 max_blocks | u64 max_in_bytes | u64 out_cap | u32 nframes | nframes x (u64 in_off | u64 in_len)
//               prints per frame "status in_off in_len bs fresh first_block slot_base ovh hdr_len", then "nblocks".
//               A frame inside capacity is also placed by fb::plan_frame after the frame before it; the driver exits
//               with 3 if the two placements differ.
//   1 (header): the five i32 info fields | u64 content_size
//               prints the header's bytes in hex.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../lz4_flex_b200/csrc/lz4b200_frame_batch.cuh"

using namespace lz4b200::fb;

static bool read_exact(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

static bool read_info(lz4b200_frame_info &info)
{
    info = lz4b200_frame_info{};
    return read_exact(&info.block_size_id, 4) && read_exact(&info.block_checksums, 4) &&
           read_exact(&info.content_checksum, 4) && read_exact(&info.has_content_size, 4) && read_exact(&info.linked, 4);
}

int main()
{
    for (;;) {
        uint32_t kind;
        if (!read_exact(&kind, 4)) break;
        lz4b200_frame_info info;
        if (!read_info(info)) return 2;
        if (kind == 1) {
            if (!read_exact(&info.content_size, 8)) return 2;
            uint8_t hdr[15];
            const uint32_t n = write_header(info, hdr, sizeof hdr);
            if (write_header(info, hdr, n - 1) != 0) return 3;             // one byte short: nothing
            for (uint32_t i = 0; i < n; i++) printf("%02x", hdr[i]);
            printf("\n");
            continue;
        }
        BatchLimits lim;
        uint32_t n;
        if (!read_exact(&lim.blocks, 8) || !read_exact(&lim.in_bytes, 8) || !read_exact(&lim.out_bytes, 8) ||
            !read_exact(&n, 4))
            return 2;
        const uint32_t tail = info.content_checksum ? 8u : 4u;
        FrameCost sum{0, 0, 0};
        FramePlace placed{0, 0, 0};
        std::vector<FramePlan> seq(n);                                     // the synchronous call's placement
        for (uint32_t f = 0; f < n; f++) {
            uint64_t off, len;
            if (!read_exact(&off, 8) || !read_exact(&len, 8)) return 2;
            FramePlan p{};
            const FrameCost c = batch_frame(p, info, off, len);
            sum.blocks = sat_add(sum.blocks, c.blocks);
            sum.in_bytes = sat_add(sum.in_bytes, c.in_bytes);
            sum.bound = sat_add(sum.bound, c.bound);
            const int32_t st = capacity_status(sum, lim);
            if (st != LZ4B200_OK) drop_frame(p);
            const FramePlace e = frame_extent(p, tail);
            place_frame(p, placed);
            placed.blocks += e.blocks; placed.slot += e.slot; placed.ovh += e.ovh;
            if (st == LZ4B200_OK) {
                seq[f] = p;
                plan_frame(seq[f], f ? &seq[f - 1] : nullptr, tail);
                if (seq[f].first_block != p.first_block || seq[f].slot_base != p.slot_base || seq[f].ovh != p.ovh)
                    return 3;
            }
            printf("%d %llu %llu %u %u %u %llu %llu %u\n", st, (unsigned long long)p.in_off,
                   (unsigned long long)p.in_len, p.bs, p.fresh, p.first_block, (unsigned long long)p.slot_base,
                   (unsigned long long)p.ovh, (unsigned)p.hdr_len);
        }
        printf("%llu\n", (unsigned long long)placed.blocks);
    }
    return 0;
}
