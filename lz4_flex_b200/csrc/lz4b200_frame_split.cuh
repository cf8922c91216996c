// lz4b200_frame_split.cuh — where each frame of concatenated LZ4 frames starts (lz4b200_frame_split_device).
//
// The split gives exactly the regions the serial decode loop (lz4b200_frame_decompress_next_device, called again at
// in + consumed) would visit: p0 = 0; frame i is fw::frame_walk over in[p_i, n), without block checksums; when that
// walk ends with status OK and p_i + consumed_i < n, p_(i+1) = p_i + consumed_i, otherwise frame i is the last.  Region
// i is [p_i, p_(i+1)), the last region [p_last, n); n == 0 has none.
//
// The chain is serial, so it is found in four phases:
//   1. candidate scan: every position whose 4 bytes are a frame, legacy or skippable magic, compacted in position order
//      (a count per tile, scan_sizes_kernel over the tiles, then each tile writes its candidates);
//   2. bounded walks: one thread per candidate walks at most kSplitHops BlockInfo words and finds its successor among
//      the candidates by binary search;
//   3. chain walk: one CTA follows the successors from position 0, streaming them through a shared-memory window, and
//      walks on serially only at a candidate whose bounded walk did not finish (a frame of more than kSplitHops blocks,
//      which the one-frame decoder walks serially too);
//   4. more candidates than the scratch holds: the chain walk walks every frame serially.
// A magic inside a payload is a false candidate.  Its walk costs at most kSplitHops hops, so the work stays within
// kSplitHops x candidates + the blocks of the frames on the chain, whatever the payloads hold.
//
// Each phase's per-thread body is an FW_FN function, so tests/cpp/frame_split_host.cpp runs the phases on the CPU.
#pragma once
#include <stdint.h>

#include "lz4b200_frame_walk.cuh"

namespace lz4b200 {
namespace fw {

constexpr uint32_t kSplitHops = 64;                // BlockInfo words a candidate's walk reads at most
constexpr uint32_t kSplitThreadBytes = 64;         // candidate positions one scan thread covers
constexpr uint32_t kSplitTile = 256 * kSplitThreadBytes;   // positions one scan CTA (256 threads) covers

// A candidate's successor code: a candidate index, or one of these.
constexpr uint32_t kSplitUnfinished = 0xffffffffu;   // the bounded walk did not reach the frame's end
constexpr uint32_t kSplitLast = 0xfffffffeu;         // the frame's region is the last one
constexpr uint32_t kSplitNoCand = 0xfffffffdu;       // the next region starts at a position that is no candidate: it
                                                     // is the last one
constexpr uint64_t kSplitMaxCandidates = 0xfffffffcull;   // candidate indices stay below the codes

FW_FN bool split_magic(uint32_t m)
{
    return m == 0x184D2204u || m == 0x184C2102u || (m & 0xFFFFFFF0u) == 0x184D2A50u;
}

// Phase 1: the candidates p in [lo, hi) of in[0, n), in order.  With `out`, the k-th goes to out[at + k] when
// at + k < cap.  Returns their count.
FW_FN uint32_t split_scan(const uint8_t *in, uint64_t n, uint64_t lo, uint64_t hi, uint64_t *out, uint64_t at,
                          uint64_t cap)
{
    if (n < 4) return 0;
    if (hi > n - 3) hi = n - 3;
    if (lo >= hi) return 0;
    uint32_t w = ((uint32_t)in[lo] << 8) | ((uint32_t)in[lo + 1] << 16) | ((uint32_t)in[lo + 2] << 24);
    uint32_t k = 0;
    for (uint64_t p = lo; p < hi; p++) {
        w = (w >> 8) | ((uint32_t)in[p + 3] << 24);              // in[p, p + 4) little-endian
        if (split_magic(w)) {
            if (out && at + k < cap) out[at + k] = p;
            k++;
        }
    }
    return k;
}

// The index of the candidate at p among pos[lo, c) (sorted), or kSplitNoCand.
FW_FN uint32_t split_find(const uint64_t *pos, uint32_t lo, uint32_t c, uint64_t p)
{
    uint32_t hi = c;
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (pos[mid] < p) lo = mid + 1; else hi = mid;
    }
    return lo < c && pos[lo] == p ? lo : kSplitNoCand;
}

// The walk of the frame at in[p, n) for at most max_hops BlockInfo words (hops, added to *hops).  Returns false when
// it did not end within them; otherwise *end is where the next region starts, or n when this frame's region is the
// last.
FW_FN bool split_frame(const uint8_t *in, uint64_t n, uint64_t p, uint64_t max_hops, uint64_t *end, uint64_t *hops)
{
    FrameWalk w;
    FrameBlockDesc buf[4];
    while (w.stage != kWalkDone && w.nblocks < max_hops) {
        const uint64_t left = max_hops - w.nblocks;
        frame_walk(in + p, n - p, w, buf, left < 4 ? (uint32_t)left : 4u);
    }
    *hops += w.nblocks;
    if (w.stage != kWalkDone) return false;
    *end = w.status == LZ4B200_OK && w.ip < n - p ? p + w.ip : n;
    return true;
}

// Phase 2: candidate i of the c at pos[]: its successor code, and in *end where its region ends when that code is a
// candidate index or kSplitNoCand.
FW_FN uint32_t split_candidate(const uint8_t *in, uint64_t n, const uint64_t *pos, uint32_t c, uint32_t i,
                               uint64_t *end, uint64_t *hops)
{
    *end = n;
    if (!split_frame(in, n, pos[i], kSplitHops, end, hops)) return kSplitUnfinished;
    if (*end == n) return kSplitLast;
    return split_find(pos, i + 1, c, *end);
}

// Phase 3: the chain walk's state.  `start` is where the next region starts and `cand` the candidate there
// (kSplitNoCand: none, so that region is the last).  `serial`: phase 4, every frame walked in full.
struct SplitChain {
    uint64_t start = 0;
    uint64_t regions = 0;
    uint32_t cand = kSplitNoCand;
    uint8_t done = 0, serial = 0;
};

// The successor codes and region ends of candidates [lo, hi), as the chain walk sees them.
struct SplitWindow {
    uint32_t lo = 0, hi = 0;
    const uint32_t *next = nullptr;
    const uint64_t *end = nullptr;
};

FW_FN void split_chain_init(SplitChain &s, uint64_t n, const uint64_t *pos, uint64_t c, uint64_t max_candidates)
{
    s = SplitChain{};
    s.done = n == 0;
    s.serial = c > max_candidates;
    if (!s.serial && c && pos[0] == 0) s.cand = 0;
}

// Writes regions (off[r], len[r]) until the input is split, max_frames regions are written, or the successor of a
// candidate outside the window is needed: then returns that candidate, which the caller loads the window from (chain
// positions only increase, so a window never needs to move back).  Sets s.done when finished.
FW_FN uint32_t split_chain(const uint8_t *in, uint64_t n, const uint64_t *pos, uint32_t c, SplitChain &s,
                           const SplitWindow &win, uint64_t *off, uint64_t *len, uint64_t max_frames, uint64_t *hops)
{
    while (!s.done) {
        if (s.regions >= max_frames) { s.done = 1; break; }
        uint64_t end = n;
        uint32_t next = kSplitLast;
        if (s.serial) {
            split_frame(in, n, s.start, ~0ull, &end, hops);
            next = end == n ? kSplitLast : kSplitNoCand;
        } else if (s.cand != kSplitNoCand) {
            if (s.cand < win.lo || s.cand >= win.hi) return s.cand;
            next = win.next[s.cand - win.lo];
            if (next == kSplitUnfinished) {                          // a long frame: walked on here
                split_frame(in, n, s.start, ~0ull, &end, hops);
                next = end == n ? kSplitLast : split_find(pos, s.cand + 1, c, end);
            } else if (next != kSplitLast) {
                end = win.end[s.cand - win.lo];
            }
        }
        off[s.regions] = s.start;
        len[s.regions] = end - s.start;
        s.regions++;
        s.start = end;
        if (next == kSplitLast) s.done = 1;
        else s.cand = next;
    }
    return kSplitNoCand;
}

}  // namespace fw
}  // namespace lz4b200
