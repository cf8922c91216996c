// Host build of the frame split (lz4_flex_b200/csrc/lz4b200_frame_split.cuh) for CPU-side tests: the per-thread bodies
// of its four phases, run one after another on the CPU the way lz4b200_frame_split_device runs them on the GPU (scan
// threads of kSplitThreadBytes positions, tiles of 256 threads, a chain walk that streams windows of 2 048 candidates),
// compiled by g++ with AddressSanitizer and UndefinedBehaviorSanitizer and driven by tests/test_frame_split_host.py.
// Test infrastructure only: nothing in the product links or runs this.
//
// stdin: records of  u64 max_frames | u64 max_candidates | u64 n | n bytes.  Every input is copied into an allocation
// of exactly n bytes, so the sanitizer reports any read past n.
// stdout per record: "regions covered candidates hops bound", then one "offset length" line per region.  hops counts
// the BlockInfo words every walk read (phases 2 to 4); bound is the sum of frame_bound_kernel's rule over the regions.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../lz4_flex_b200/csrc/lz4b200_frame_split.cuh"

using namespace lz4b200::fw;

static bool read_exact(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

int main()
{
    for (;;) {
        uint64_t max_frames, max_cand, n;
        if (!read_exact(&max_frames, 8)) break;
        if (!read_exact(&max_cand, 8) || !read_exact(&n, 8)) return 2;
        uint8_t *buf = (uint8_t *)malloc(n ? n : 1);
        if (n && !read_exact(buf, n)) return 2;
        const uint8_t *in = n ? buf : nullptr;

        // phase 1: per-thread counts, tile offsets, then each thread writes its candidates
        const uint64_t threads = (n + kSplitThreadBytes - 1) / kSplitThreadBytes;
        std::vector<uint32_t> count(threads);
        uint64_t total = 0;
        for (uint64_t t = 0; t < threads; t++) {
            count[t] = split_scan(in, n, t * kSplitThreadBytes, (t + 1) * kSplitThreadBytes, nullptr, 0, 0);
            if (count[t] > 16) return 3;
            total += count[t];
        }
        std::vector<uint64_t> pos(max_cand ? max_cand : 1);
        uint64_t at = 0;
        for (uint64_t t = 0; t < threads; t++) {
            if (count[t])
                split_scan(in, n, t * kSplitThreadBytes, (t + 1) * kSplitThreadBytes, pos.data(), at, max_cand);
            at += count[t];
        }

        // phase 2: the bounded walks, when the candidates fit
        uint64_t hops = 0;
        const uint32_t c = total > max_cand ? 0u : (uint32_t)total;
        std::vector<uint32_t> next(c ? c : 1);
        std::vector<uint64_t> end(c ? c : 1);
        for (uint32_t i = 0; i < c; i++) {
            uint64_t h = 0;
            next[i] = split_candidate(in, n, pos.data(), c, i, &end[i], &h);
            if (h > kSplitHops) return 4;
            hops += h;
        }

        // phases 3 and 4: the chain walk over windows of 2 048 candidates, each loaded once, in increasing order
        const uint64_t slots = (max_frames < n ? max_frames : n) + 1;          // a region holds at least one byte
        std::vector<uint64_t> off(slots), len(slots);
        SplitChain st;
        SplitWindow win;
        split_chain_init(st, n, pos.data(), total, max_cand);
        int64_t last_lo = -1;
        for (;;) {
            const uint32_t need = split_chain(in, n, pos.data(), c, st, win, off.data(), len.data(), max_frames, &hops);
            if (st.done) break;
            if ((int64_t)need <= last_lo || need >= c) return 5;
            last_lo = need;
            win.lo = need;
            win.hi = (uint64_t)need + 2048 < c ? need + 2048 : c;
            win.next = next.data() + need;
            win.end = end.data() + need;
        }

        // frame_bound_kernel's rule per region, summed
        uint64_t bound = 0;
        for (uint64_t r = 0; r < st.regions; r++) {
            FrameWalk w;
            FrameBlockDesc b[4];
            while (w.stage != kWalkDone) {
                const uint32_t k = frame_walk(in + off[r], len[r], w, b, 4);
                for (uint32_t i = 0; i < k; i++)
                    bound += block_stored(b[i]) ? block_len(b[i]) : block_decoded_cap(block_len(b[i]), w.bs);
            }
        }
        printf("%llu %llu %llu %llu %llu\n", (unsigned long long)st.regions, (unsigned long long)st.start,
               (unsigned long long)total, (unsigned long long)hops, (unsigned long long)bound);
        for (uint64_t r = 0; r < st.regions; r++)
            printf("%llu %llu\n", (unsigned long long)off[r], (unsigned long long)len[r]);
        free(buf);
    }
    return 0;
}
