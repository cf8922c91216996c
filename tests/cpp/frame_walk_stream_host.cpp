// Host build of the streaming frame walk (fw::frame_walk_stream, lz4_flex_b200/csrc/lz4b200_frame_walk.cuh) for CPU-side
// tests, compiled by g++ with AddressSanitizer and UndefinedBehaviorSanitizer and driven by
// tests/test_frame_walk_stream_host.py.  Test infrastructure only: nothing in the product links or runs this.
//
// stdin: records of  u32 max_blocks | u64 n | n bytes | u32 nsplit | nsplit x u64 split.  The splits are increasing
// ends of the input available so far; the last is n, and it is presented with eof.  Each call gets an allocation of
// exactly the bytes it is presented, from the walk's position to the current split, so the sanitizer reports any read
// at or past its n.  The walk is called with the same bytes until it stops making progress, then the next split comes.
//
// stdout, one line per record:  "<ok> <status> <ip> <nblocks> <calls>"  where ok is 1 when the streaming walk recorded
// the blocks frame_walk records on the whole input, at the same frame offsets, and ended in the same FrameWalk; it is 0
// otherwise, or when a call broke a rule: a stop for input left a status, a `need` not past the bytes presented, or a
// position that is not a unit boundary of the whole-input walk.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <set>
#include <vector>

#include "../../lz4_flex_b200/csrc/lz4b200_frame_walk.cuh"

using namespace lz4b200::fw;

static bool read_exact(void *p, size_t n) { return fread(p, 1, n, stdin) == n; }

static bool same_walk(const FrameWalk &a, const FrameWalk &b)
{
    return a.ip == b.ip && a.bs == b.bs && a.content_size == b.content_size && a.nblocks == b.nblocks &&
           a.status == b.status && a.stage == b.stage && a.flg == b.flg && a.content_checksum == b.content_checksum &&
           a.has_size == b.has_size && a.has_checksum == b.has_checksum && a.closed == b.closed && a.linked == b.linked;
}

int main()
{
    for (;;) {
        uint32_t max_blocks, nsplit;
        uint64_t n;
        if (!read_exact(&max_blocks, 4)) break;
        if (!read_exact(&n, 8)) return 2;
        std::vector<uint8_t> frame(n);
        if (n && !read_exact(frame.data(), n)) return 2;
        if (!read_exact(&nsplit, 4)) return 2;
        std::vector<uint64_t> split(nsplit);
        if (nsplit && !read_exact(split.data(), nsplit * 8)) return 2;
        if (!nsplit || split.back() != n || max_blocks == 0) return 2;

        // the whole-input walk and its unit boundaries
        FrameWalk whole;
        std::vector<FrameBlockDesc> want;
        const uint8_t *all = n ? frame.data() : nullptr;
        while (whole.stage != kWalkDone) {
            const size_t at = want.size();
            want.resize(at + 4096);
            want.resize(at + frame_walk(all, n, whole, want.data() + at, 4096));
        }
        std::set<uint64_t> bounds = {0, whole.ip};
        {
            FrameWalk h;
            walk_header(all, n, h);
            bounds.insert(h.ip);
        }
        for (const FrameBlockDesc &b : want) bounds.insert(b.payload_off + block_len(b) + ((whole.flg & 0x10) ? 4 : 0));

        FrameWalk w;
        std::vector<FrameBlockDesc> got;
        bool ok = true;
        uint32_t calls = 0;
        for (uint32_t s = 0; s < nsplit && w.stage != kWalkDone; s++) {
            const bool eof = s + 1 == nsplit;
            for (;;) {
                if (split[s] < w.ip) { ok = false; break; }
                const uint64_t avail = split[s] - w.ip;
                uint8_t *buf = avail ? (uint8_t *)malloc(avail) : nullptr;
                if (avail) memcpy(buf, frame.data() + w.ip, avail);
                const uint64_t at = w.ip, before = w.nblocks;
                std::vector<FrameBlockDesc> out(std::min<uint64_t>(max_blocks, avail / 4 + 1));   // a block takes >= 4 bytes
                uint64_t need = 0;
                const uint32_t k = frame_walk_stream(buf, avail, eof, w, out.data(), (uint32_t)out.size(), &need);
                free(buf);
                calls++;
                if (w.nblocks != before + k) ok = false;
                for (uint32_t i = 0; i < k; i++) {
                    out[i].payload_off += at;
                    got.push_back(out[i]);
                }
                if (!bounds.count(w.ip)) ok = false;
                if (need) {
                    if (eof || w.stage == kWalkDone || w.status != LZ4B200_OK || need <= split[s] - w.ip || need < 4) ok = false;
                    break;
                }
                if (w.stage == kWalkDone) break;
                if (k == 0 && w.ip == at) { ok = false; break; }     // neither stopped for input nor made progress
            }
            if (!ok) break;
        }
        ok = ok && w.stage == kWalkDone && same_walk(w, whole) && got.size() == want.size();
        for (size_t i = 0; ok && i < got.size(); i++)
            ok = got[i].payload_off == want[i].payload_off && got[i].word == want[i].word && got[i].checksum == want[i].checksum;
        printf("%d %d %llu %llu %u\n", ok ? 1 : 0, w.status, (unsigned long long)w.ip, (unsigned long long)w.nblocks, calls);
    }
    return 0;
}
