// Host build of the streaming frame encoder's plan (lz4_flex_b200/csrc/lz4b200_frame_encoder.cuh): where each call cuts
// blocks and groups, each block's parse mode and stream offset, the header and EndMark, and the call's bound, compiled
// by g++ with AddressSanitizer and UndefinedBehaviorSanitizer and driven by tests/test_frame_encoder_host.py.  Test
// infrastructure only: nothing in the product links or runs this.
//
// stdin: records of  u32 nops | i32 block_size_id | u8 block_checksums | u8 content_checksum | u8 has_content_size |
//                    u64 content_size | u64 budget, then nops x (u64 n | u8 op).
// Each call prints "status header endmark block_size_id group bound nsteps nblocks buffered content_len" (the last two
// after the call), then per step "src dst len group_len nblocks b0" (b0: the call's blocks before the step's group), then
// per block "flags stream_offset", the flags being what fb::batch_block gives the block in its step's group_plan.
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../lz4_flex_b200/csrc/lz4b200_frame_encoder.cuh"

using namespace lz4b200::fe;

static bool read_exact(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main()
{
    for (;;) {
        uint32_t nops;
        if (!read_exact(&nops, 4)) break;
        lz4b200_frame_info info{};
        uint8_t bc, cc, hs;
        uint64_t budget;
        if (!read_exact(&info.block_size_id, 4) || !read_exact(&bc, 1) || !read_exact(&cc, 1) || !read_exact(&hs, 1) ||
            !read_exact(&info.content_size, 8) || !read_exact(&budget, 8))
            return 2;
        info.block_checksums = bc;
        info.content_checksum = cc;
        info.has_content_size = hs;
        State s;
        s.block_size_id = info.block_size_id;
        for (uint32_t i = 0; i < nops; i++) {
            uint64_t n;
            uint8_t op;
            if (!read_exact(&n, 8) || !read_exact(&op, 1)) return 2;
            const uint64_t bound = call_bound(s, info, budget, n, op);
            const CallPlan p = plan_call(s, info, budget, n, op);
            printf("%d %u %u %d %llu %llu %zu %zu %llu %llu\n", p.status, (unsigned)p.header, (unsigned)p.endmark,
                   p.block_size_id, (unsigned long long)p.group, (unsigned long long)bound, p.steps.size(),
                   p.block_off.size(), (unsigned long long)p.next.buffered, (unsigned long long)p.next.content_len);
            std::vector<uint8_t> flags;
            for (const Step &st : p.steps) {
                printf("%llu %llu %llu %llu %u %zu\n", (unsigned long long)st.src, (unsigned long long)st.dst,
                       (unsigned long long)st.len, (unsigned long long)st.group_len, st.nblocks, flags.size());
                if (!st.group_len) continue;
                const lz4b200::fb::FramePlan g = group_plan(st, block_bytes(p.block_size_id));
                for (uint32_t k = 0; k < st.nblocks; k++) flags.push_back(lz4b200::fb::batch_block(&g, 1, k).flags);
            }
            if (flags.size() != p.block_off.size()) return 3;
            for (size_t b = 0; b < flags.size(); b++)
                printf("%u %llu\n", (unsigned)flags[b], (unsigned long long)p.block_off[b]);
            s = p.next;
        }
    }
    return 0;
}
