// Host build of the batch frame encoder's plan (lz4_flex_b200/csrc/lz4b200_frame_batch.cuh): the per-frame plan, the
// per-block mapping and the frames' places in the packed output, compiled by g++ with AddressSanitizer and
// UndefinedBehaviorSanitizer and driven by tests/test_frame_batch_host.py.  Test infrastructure only: nothing in the
// product links or runs this.
//
// stdin: records of  u32 nframes | u32 tail_len |
//                    nframes x (u64 in_off | u64 in_len | u32 bs | u32 fresh | u32 first_fresh | u8 hdr_len)
//        followed by one u32 segment size per block of the batch.
// Each record prints "nblocks slots", then per block "frame k in_off in_len out_off out_cap flags dst" (dst: the
// segment's offset in the packed output), then per frame "start endmark".
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../lz4_flex_b200/csrc/lz4b200_frame_batch.cuh"

using namespace lz4b200::fb;

static bool read_exact(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main()
{
    for (;;) {
        uint32_t n, tail;
        if (!read_exact(&n, 4)) break;
        if (!read_exact(&tail, 4)) return 2;
        std::vector<FramePlan> plan(n);
        uint64_t nb = 0, slots = 0;
        for (uint32_t f = 0; f < n; f++) {
            FramePlan &p = plan[f];
            if (!read_exact(&p.in_off, 8) || !read_exact(&p.in_len, 8) || !read_exact(&p.bs, 4) ||
                !read_exact(&p.fresh, 4) || !read_exact(&p.first_fresh, 4) || !read_exact(&p.hdr_len, 1))
                return 2;
            plan_frame(p, f ? &plan[f - 1] : nullptr, tail);
            nb += frame_blocks(p);
            slots += frame_slot_bytes(p);
        }
        std::vector<uint32_t> seg(nb);
        std::vector<uint64_t> seg_off(nb + 1, 0);
        if (nb && !read_exact(seg.data(), 4 * nb)) return 2;
        for (uint64_t b = 0; b < nb; b++) seg_off[b + 1] = seg_off[b] + seg[b];
        printf("%llu %llu\n", (unsigned long long)nb, (unsigned long long)slots);
        for (uint32_t b = 0; b < (uint32_t)nb; b++) {
            const BlockJob j = batch_block(plan.data(), n, b);
            printf("%u %u %llu %u %llu %u %u %llu\n", j.frame, j.k, (unsigned long long)j.in_off, j.in_len,
                   (unsigned long long)j.out_off, j.out_cap, (unsigned)j.flags,
                   (unsigned long long)(seg_off[b] + j.dst_shift));
        }
        for (uint32_t f = 0; f < n; f++) {
            uint64_t start, endmark;
            frame_place(plan[f], seg_off.data(), &start, &endmark);
            printf("%llu %llu\n", (unsigned long long)start, (unsigned long long)endmark);
        }
    }
    return 0;
}
