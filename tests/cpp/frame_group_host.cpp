// Host build of the batch frame decoder's planning step (lz4_flex_b200/csrc/lz4b200_frame_walk.cuh): the count walk
// and the group loop's cut that the one-frame group loop and the batch decoder share, compiled by g++ with
// AddressSanitizer and UndefinedBehaviorSanitizer and driven by tests/test_frame_group_host.py.  Test infrastructure
// only: nothing in the product links or runs this.
//
// stdin: records of  u8 op | u64 budget | ...
//   op 0: u64 bs | u32 nblocks | nblocks x (u64 payload_off | u32 word): frame_count_add over the list;
//   op 1: u64 n | n bytes (an allocation of exactly n bytes): frame_count over the frame.
// Each record prints "slot_total nblocks one_group linked status consumed" (status and consumed: op 1 only, else 0).
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../lz4_flex_b200/csrc/lz4b200_frame_walk.cuh"

using namespace lz4b200::fw;

static bool read_exact(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main()
{
    for (;;) {
        uint8_t op;
        uint64_t budget;
        if (!read_exact(&op, 1)) break;
        if (!read_exact(&budget, 8)) return 2;
        FrameCount c;
        FrameWalk w;
        if (op == 0) {
            uint64_t bs;
            uint32_t nb;
            if (!read_exact(&bs, 8) || !read_exact(&nb, 4)) return 2;
            for (uint32_t k = 0; k < nb; k++) {
                FrameBlockDesc b{};
                if (!read_exact(&b.payload_off, 8) || !read_exact(&b.word, 4)) return 2;
                frame_count_add(c, b, bs, budget);
            }
        } else {
            uint64_t n;
            if (!read_exact(&n, 8)) return 2;
            uint8_t *buf = (uint8_t *)malloc(n ? n : 1);
            if (n && !read_exact(buf, n)) return 2;
            frame_count(n ? buf : nullptr, n, w, c, budget);
            free(buf);
        }
        printf("%llu %llu %d %d %d %llu\n", (unsigned long long)c.slot_total, (unsigned long long)c.nblocks,
               (int)c.one_group, (int)c.linked, w.status, (unsigned long long)w.ip);
    }
    return 0;
}
