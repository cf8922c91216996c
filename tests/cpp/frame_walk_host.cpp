// Host build of the frame walk and XXH32 (lz4_flex_b200/csrc/lz4b200_frame_walk.cuh) for CPU-side tests: the code the
// device walk kernel and lz4b200_frame_decompress_next both run, compiled by g++ with AddressSanitizer and
// UndefinedBehaviorSanitizer and driven by tests/test_frame_walk_host.py.  Test infrastructure only: nothing in the
// product links or runs this.
//
// stdin: records of  u8 op | u32 arg | u64 n | n bytes.  Every input is copied into an allocation of exactly n bytes,
// so the sanitizer reports any read past n.
//   op 0: XXH32 with seed `arg`, printed one-shot and streamed in pieces of 1, 5, 16 and 33 bytes;
//   op 1: the frame walk, `arg` blocks per frame_walk() call (the device walk resumes launch after launch the same
//         way), then the block checksum step; prints "status consumed nblocks flg closed" and one
//         "payload_off word checksum" line per block.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../lz4_flex_b200/csrc/lz4b200_frame_walk.cuh"

using namespace lz4b200::fw;

static bool read_exact(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

static uint32_t xxh32_pieces(const uint8_t *p, uint64_t n, uint32_t seed, uint64_t piece)
{
    lz4b200_xxh32_state st;
    xxh32_reset(st, seed);
    for (uint64_t o = 0; o < n; o += piece) xxh32_update(st, p + o, n - o < piece ? n - o : piece);
    return xxh32_digest(st);
}

int main()
{
    for (;;) {
        uint8_t op;
        uint32_t arg;
        uint64_t n;
        if (!read_exact(&op, 1)) break;
        if (!read_exact(&arg, 4) || !read_exact(&n, 8)) return 2;
        uint8_t *buf = (uint8_t *)malloc(n ? n : 1);
        if (n && !read_exact(buf, n)) return 2;
        const uint8_t *in = n ? buf : nullptr;
        if (op == 0) {
            printf("%u %u %u %u %u\n", xxh32(in, n, arg), xxh32_pieces(in, n, arg, 1), xxh32_pieces(in, n, arg, 5),
                   xxh32_pieces(in, n, arg, 16), xxh32_pieces(in, n, arg, 33));
        } else {
            FrameWalk w;
            std::vector<FrameBlockDesc> blocks;
            while (w.stage != kWalkDone) {
                const size_t at = blocks.size();
                blocks.resize(at + arg);
                blocks.resize(at + frame_walk(in, n, w, blocks.data() + at, arg));
            }
            if (blocks.size() != w.nblocks) return 3;
            if (w.flg & 0x10) {
                for (size_t k = 0; k < blocks.size(); k++)
                    if (!block_checksum_ok(in, blocks[k])) {
                        frame_walk_fail_block(w, blocks[k], (uint32_t)k);
                        blocks.resize(k);
                        break;
                    }
            }
            printf("%d %llu %zu %u %d\n", w.status, (unsigned long long)w.ip, blocks.size(), w.flg, (int)w.closed);
            for (const FrameBlockDesc &b : blocks)
                printf("%llu %u %u\n", (unsigned long long)b.payload_off, b.word, b.checksum);
        }
        free(buf);
    }
    return 0;
}
