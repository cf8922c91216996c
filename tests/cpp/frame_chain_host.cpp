// Host build of the linked frame's per-block plan (lz4_flex_b200/csrc/lz4b200_frame_chain.cuh), compiled by g++ with
// AddressSanitizer and UndefinedBehaviorSanitizer and driven by tests/test_frame_linked_compress.py.  Test
// infrastructure only: nothing in the product links or runs this.
//
// stdin: records of  u64 bs | u64 stream | u64 ext_len | u64 src_start | u32 nblocks | nblocks x u64 length
//        (stream, ext_len and src_start set the state before the first block; all 0 for a frame's start).
// Each record prints one line per block: "stream ext_len prefix reposition shift to_frame first".
#include <cstdint>
#include <cstdio>
#include <vector>

#include "../../lz4_flex_b200/csrc/lz4b200_frame_chain.cuh"

using namespace lz4b200::fb;

static bool read_exact(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main()
{
    for (;;) {
        uint64_t bs, stream, ext, start;
        uint32_t n;
        if (!read_exact(&bs, 8)) break;
        if (!read_exact(&stream, 8) || !read_exact(&ext, 8) || !read_exact(&start, 8) || !read_exact(&n, 4)) return 2;
        std::vector<uint64_t> len(n);
        if (n && !read_exact(len.data(), 8 * n)) return 2;
        ChainState c = chain_start(bs);
        c.stream = stream; c.ext_len = ext; c.src_start = start; c.consumed = start;
        for (uint32_t k = 0; k < n; k++) {
            const ChainBlock b = chain_next(c, len[k]);
            printf("%llu %u %u %d %llu %lld %d\n", (unsigned long long)b.stream, b.ext_len, b.prefix, (int)b.reposition,
                   (unsigned long long)b.shift, (long long)b.to_frame, (int)b.first);
        }
    }
    return 0;
}
