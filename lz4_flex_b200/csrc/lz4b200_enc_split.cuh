// lz4b200_enc_split.cuh — K1 as a matcher/emitter warp pipeline (included by lz4b200_kernels.cuh).
//
// Two kernels share the code below: lz4_compress_blocks_split (one emitter per matcher, tables in shared memory,
// 24 matchers per SM) and lz4_compress_blocks_gtab (7 matchers per emitter, each table in shared memory or in global
// memory served by L2; 21 matchers per SM by default, all with shared-memory tables).  The launcher picks by batch
// size (DESIGN.md §4).
//
// compress_internal (reference src/block/compress.rs:318-489) does two things per sequence: it SEARCHES
// (probe loop :373-439, backward/forward extension :272-287 / :156-216, the cur-2 re-insert :460-461) and it
// EMITS (token, length bytes, literals, offset: :463-486).  Only the search is a serial chain — the next
// probe starts where this match ends — while emission depends on nothing but the finished
// (anchor, match start, offset, match end) tuple.  So a block is handled by a PAIR of warps:
//
//   matcher warp : owns the block's 4096-slot table and runs the exact emulation of the sequential probe loop
//                  (32 probes per batch, speculative pre-batch candidates, in-batch table forwarding with
//                  shuffles / match.any only when slots collide); it pushes one 16-byte tuple per sequence into a
//                  shared-memory ring and goes straight on to the next probe.
//   emitter warp : takes a batch of tuples at a time, one per lane; every lane sizes its own sequence, a warp
//                  exclusive scan (__shfl_up) turns sizes into output offsets, and the lanes write token /
//                  length bytes / literals / offset of the whole batch at once (long literal runs are copied by the
//                  whole warp).  This is the scan-compacted emission the north star asks for, and it takes
//                  ~27 % of the per-sequence chain off the matcher (DESIGN.md §6).
//
// Hand-off: two halves of 16 tuples, mbarriers "full[h]" / "empty[h]" per pair in shared memory — the matcher
// never waits unless the emitter is two batches behind.
#pragma once
#ifndef ENC_GTAB_L1
#define ENC_GTAB_L1 0   // 1: global-table reads may hit L1 (same-SM coherent); 0: L2 only
#endif
#ifndef ENC_FIRST_WIDTH
#define ENC_FIRST_WIDTH 32  // lanes probing in the first round of a sequence (8 was slower: the extra round costs more than the traffic it saves)
#endif
#ifndef ENC_FASTW
#define ENC_FASTW 1     // 1: settle slot collisions of the first <= 4 probes with shuffles instead of match.any
#endif
#ifndef ENC_RI_PATCH
#define ENC_RI_PATCH 0  // 1: re-insert folded into the batch commit (no store->load dependency); 0: store + syncwarp first
#endif
#ifndef ENC_EMIT_SLEEP_NS
#define ENC_EMIT_SLEEP_NS 1000   // emitter back-off while its queue is empty (0: spin)
#endif
#ifndef ENC_WINDOW
#define ENC_WINDOW 0   // 1: first probe batch reads a cp.async-filled shared-memory ring (measured slightly slower)
#endif

namespace lz4b200 {

#ifndef ENC_SEQ_BATCH
#define ENC_SEQ_BATCH 16   // tuples per hand-off (1..32): the emitter's cost per batch does not depend on it
#endif
constexpr uint32_t kSeqBatchEntries = ENC_SEQ_BATCH;      // tuples per hand-off (two halves per ring)
constexpr uint32_t kWinBytes = 512;            // input look-ahead ring per pair: 4 lines of 128 bytes
constexpr uint32_t kRingBytes = ENC_WINDOW ? kWinBytes : 0;   // shared memory actually reserved for it
constexpr uint32_t kExitBlock = 0xffffffffu;
constexpr uint32_t kSmallLit = 24;            // literal runs up to this length are copied by the owning lane

#ifdef LZ4B200_ENC_PROFILE
// Development build only (tests/dev/enc_phase_probe.py; neither library defines it): the matcher's clock64() cycles per phase
// of match_block_view and a few event counts, kept per block in registers and added to g_enc_profile by lane 0 when the
// block ends.  The cycles of a phase run from the end of the previous phase to the first warp-wide step that consumes its
// results, so a load's latency is charged to the phase that waits for it.
enum EncProfSlot : int {
    kPhProbe,      // probe batch: re-insert, input and table loads, candidate fetch, hit ballot
    kPhResolve,    // in-batch slot collisions (shuffles / match.any) and the forwarded candidates
    kPhCommit,     // table writes of the executed probes, winner broadcast, next batch set-up
    kPhExtend,     // backward and forward extension
    kPhPush,       // tuple hand-off, including the wait for a free ring half
    kPhSetup,      // table reset and the first insert of a block
    kCtSeq,        // sequences (tuples with a match)
    kCtBatch,      // probe batches
    kCtNoBack,     // sequences without literals before the match (no backward round)
    kCtShort,      // sequences with no backward round whose forward mismatch is within 8 bytes of the match start + 4
    kCtLong,       // sequences that needed a second forward round (match longer than 36 bytes)
    kCtBlocks,     // blocks
    kEncProfSlots = 16
};
__device__ unsigned long long g_enc_profile[kEncProfSlots];
struct EncProfile {
    uint64_t t;
    uint32_t c[kEncProfSlots];
    __device__ __forceinline__ void start()
    {
#pragma unroll
        for (int i = 0; i < kEncProfSlots; i++) c[i] = 0;
        t = clock64();
    }
    __device__ __forceinline__ void phase(int i) { const uint64_t now = clock64(); c[i] += (uint32_t)(now - t); t = now; }
    __device__ __forceinline__ void count(int i, bool on = true) { c[i] += on ? 1u : 0u; }
    __device__ __forceinline__ void flush(uint32_t lane)
    {
        c[kCtBlocks]++;
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < kEncProfSlots; i++)
                if (c[i]) atomicAdd(g_enc_profile + i, (unsigned long long)c[i]);
        }
    }
};
#define ENC_PROF(x) prof.x
#else
#define ENC_PROF(x) ((void)0)
#endif

// mbarrier hand-off (shared-memory barrier objects; named barriers would cost 16 hardware barriers per CTA
// and cap the resident CTAs).  One arrival per phase, from lane 0 of the signalling warp, after its writes.
__device__ __forceinline__ uint32_t smem_addr(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_addr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar)
{
    asm volatile("{ .reg .b64 st; mbarrier.arrive.release.cta.shared::cta.b64 st, [%0]; }" ::"r"(smem_addr(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    const uint32_t addr = smem_addr(bar);
    uint32_t done;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    } while (!done);
}
// Producer-side wait for a free ring half.  One emitter serves 7 matchers, so a matcher finds its half still unread
// every few batches; spinning there cost about a seventh of the kernel's warp-instructions (YIELD / try_wait / BRA) in a
// kernel that is bound by instruction issue.
// One immediate probe (the common case: already free), then try_wait with a suspend hint + nanosleep.
#ifndef ENC_PROD_SLEEP_NS
#define ENC_PROD_SLEEP_NS 200   // 0: spin (round-1 behaviour)
#endif
__device__ __forceinline__ void mbar_wait_producer(uint64_t *bar, uint32_t parity)
{
#if ENC_PROD_SLEEP_NS == 0
    mbar_wait(bar, parity);
#else
    const uint32_t addr = smem_addr(bar);
    uint32_t done;
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    while (!done) {
        __nanosleep(ENC_PROD_SLEEP_NS);
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2, %3; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(addr), "r"(parity), "r"(4u * ENC_PROD_SLEEP_NS) : "memory");
    }
#endif
}
// Consumer-side wait: the emitter is idle most of the time; spinning on try_wait would burn issue slots the
// matchers need, so it backs off between polls.
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t *bar, uint32_t parity)
{
    const uint32_t addr = smem_addr(bar);
    for (;;) {
        uint32_t done;
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2, %3; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(addr), "r"(parity), "r"(4u * ENC_EMIT_SLEEP_NS) : "memory");
        if (done) break;
#if ENC_EMIT_SLEEP_NS
        __nanosleep(ENC_EMIT_SLEEP_NS);
#endif
    }
}

// Producer side of the tuple ring (all state is warp-uniform).
struct SeqProducer {
    uint4 *q;                 // [2][32] tuples: (anchor, match start, offset, match end); offset 0 = last literals
    volatile uint32_t *meta;  // [2][4]: block index, tuple count, flags (1 = first batch of the block, 2 = last)
    uint64_t *bars;           // full[0], full[1], empty[0], empty[1]
    uint32_t k;               // batches handed over so far
    uint32_t qn;              // tuples in the current half
    uint32_t block;
    uint32_t first;

    __device__ __forceinline__ void flush(uint32_t last, uint32_t lane)
    {
        const uint32_t h = k & 1u;
        if (lane == 0) {
            meta[h * 4 + 0] = block;
            meta[h * 4 + 1] = qn;
            meta[h * 4 + 2] = first | (last << 1);
            mbar_arrive(bars + h);                             // release: tuples + header visible to the emitter
        }
        k++; qn = 0; first = 0;
        // batch k goes into half k&1, last used by batch k-2: wait until the emitter has read it
        if (k >= 2) mbar_wait_producer(bars + 2 + (k & 1u), ((k >> 1) - 1u) & 1u);
        __syncwarp();
    }
    __device__ __forceinline__ void push(uint32_t anchor, uint32_t mpos, uint32_t dist, uint32_t end, uint32_t lane)
    {
        if (lane == 0) q[(k & 1u) * kSeqBatchEntries + qn] = make_uint4(anchor, mpos, dist, end);
        qn++;
        if (qn == kSeqBatchEntries) flush(0, lane);
    }
    // the last tuple of a block (literals only): hand the batch over with the "last" flag
    __device__ __forceinline__ void push_final(uint32_t anchor, uint32_t n, uint32_t lane)
    {
        if (lane == 0) q[(k & 1u) * kSeqBatchEntries + qn] = make_uint4(anchor, 0u, 0u, n);
        qn++;
        flush(1, lane);
    }
};

// ---------------------------------------------------------------------------------------------
// Input look-ahead window.  With 24 tables resident per SM the L1 is down to its 28 KB floor, so every
// global load is an L2 round trip (several hundred cycles under load) and the probe loop would pay one per
// sequence just to read the bytes at the cursor.  Instead the matcher keeps the four 128-byte lines
// [c-1, c+3) around the cursor (c = line of the cursor) in a shared-memory ring, filled by asynchronous
// global->shared copies (cp.async, 16 bytes per lane, L2-only) that are issued two lines ahead of their
// first use.  The first probe batch (32 probes, <= 40 bytes), the re-insert of cur-2 and the input side of
// the first forward-extension round read the ring (29-cycle LDS); only the candidate side goes to L2.
// Positions are kept in "x space": x = position + (src & 127), so ring lines are 128-byte aligned in memory
// and every 16-byte copy is aligned.  Copies are clipped to the block: a chunk that ends before the block or
// starts after it reads nothing (src-size 0 = zero fill), the last chunk reads only the block's bytes.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(uint32_t saddr, const void *g, uint32_t bytes)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(saddr), "l"(g), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

struct InputWindow {
    const uint32_t *ring;     // kWinBytes / 4 words
    uint32_t ring_s;          // shared-space address of the ring
    const uint8_t *src_al;    // src rounded down to 128 bytes
    uint32_t mis;             // src - src_al
    uint32_t xend;            // mis + n
    uint32_t nlines;          // lines that contain block bytes
    uint32_t hi;              // lines below hi have been requested
    uint32_t ready;           // lines below ready have landed

    __device__ __forceinline__ void init(const uint8_t *src, uint32_t n, uint32_t *ring_)
    {
        ring = ring_;
        ring_s = smem_addr(ring_);
        mis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 127u);
        src_al = src - mis;
        xend = mis + n;
        nlines = (xend + 127u) >> 7;
        hi = 0; ready = 0;
    }
    // Request the lines of [c-1, c+3) that are not resident yet and make sure those needed now have landed.
    __device__ __forceinline__ void advance(uint32_t xc, uint32_t lane)
    {
        const uint32_t c = xc >> 7;
        const uint32_t want = min(c + 3u, nlines);
        if (hi < want) {
            const uint32_t first = max(hi, c ? c - 1u : 0u);
            const uint32_t line = first + (lane >> 3);
            if (line < want) {
                const uint32_t xo = line * 128u + (lane & 7u) * 16u;
                uint32_t bytes = 0;
                if (xo + 16u > mis && xo < xend) bytes = min(16u, xend - xo);
                cp_async16(ring_s + (xo & (kWinBytes - 1u)), src_al + xo, bytes);
            }
            cp_async_commit();
            hi = want;
        }
        const uint32_t need = min(((xc + 71u) >> 7) + 1u, hi);   // first batch + first extension round: < 72 bytes ahead
        if (ready < need) {
            cp_async_wait_all();
            __syncwarp();
            ready = hi;
        }
    }
    // low 5 bytes at x (ring must hold the line(s)): (lo32, hi8)
    __device__ __forceinline__ void ro5(uint32_t x, uint32_t &lo, uint32_t &hi8) const
    {
        const uint32_t a = ring[(x >> 2) & (kWinBytes / 4 - 1u)], b = ring[((x >> 2) + 1u) & (kWinBytes / 4 - 1u)];
        const uint32_t sh = (x & 3u) * 8u;
        lo = __funnelshift_r(a, b, sh);
        hi8 = (b >> sh) & 0xffu;
    }
    __device__ __forceinline__ uint8_t byte(uint32_t x) const
    {
        return reinterpret_cast<const uint8_t *>(ring)[x & (kWinBytes - 1u)];
    }
};

// ---------------------------------------------------------------------------------------------
// matcher: the search half of compress_internal.  Table semantics identical to encode_block_v1.
// ---------------------------------------------------------------------------------------------
// Table accessors.  kGT = false: the table lives in shared memory (plain indexing, LDS/STS).  kGT = true: it lives
// in global memory and is read/written through L2 (ld/st.global.cg): ~250 cycles instead of 29 per access, but no
// shared memory per matcher, so the matchers per SM are bounded by warps and registers instead of by 8 KiB tables.
// Global tables are accessed with an L2 evict_last policy (createpolicy is a constant: it folds into the access
// descriptor): the tables (8 KiB per chain) should stay resident in L2 while the input streams through it.
// With 32 registers per thread the compiler re-derives a chain's table pointer from blockIdx / threadIdx and rebuilds the
// createpolicy descriptor (5 uniform instructions) at every table access, in kernels that are bound by instruction issue:
//   ENC_TAB_OPAQUE = 1: the chain's table offset lives in one opaque 32-bit register (faster)
//   ENC_POLICY_HOIST = 1: createpolicy may be hoisted (uniform registers)
//   ENC_POLICY_HOIST = 2: u16 table accesses without the evict_last hint (fastest: the hint was neutral)
#ifndef ENC_POLICY_HOIST
#define ENC_POLICY_HOIST 2
#endif
#ifndef ENC_TAB_OPAQUE
#define ENC_TAB_OPAQUE 1
#endif
__device__ __forceinline__ uint64_t l2_keep_policy()
{
    uint64_t pol;
#if ENC_POLICY_HOIST
    asm("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
#else
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
#endif
    return pol;
}
template <bool kGT>
__device__ __forceinline__ uint32_t tab_get(const uint16_t *tab, uint32_t slot)
{
    if constexpr (kGT) {
        uint16_t v;
#if ENC_GTAB_L1
        asm volatile("ld.global.ca.L2::cache_hint.u16 %0, [%1], %2;" : "=h"(v) : "l"(tab + slot), "l"(l2_keep_policy()) : "memory");
#elif ENC_POLICY_HOIST == 2
        asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(v) : "l"(tab + slot) : "memory");
#else
        asm volatile("ld.global.cg.L2::cache_hint.u16 %0, [%1], %2;" : "=h"(v) : "l"(tab + slot), "l"(l2_keep_policy()) : "memory");
#endif
        return v;
    } else return tab[slot];
}
template <bool kGT>
__device__ __forceinline__ uint32_t tab_get(const uint32_t *tab, uint32_t slot)
{
    if constexpr (kGT) {
        uint32_t v;
        asm volatile("ld.global.cg.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(tab + slot), "l"(l2_keep_policy()) : "memory");
        return v;
    } else return tab[slot];
}
template <bool kGT>
__device__ __forceinline__ void tab_put(uint16_t *tab, uint32_t slot, uint32_t v)
{
    if constexpr (kGT) {
#if ENC_POLICY_HOIST == 2
        asm volatile("st.global.cg.u16 [%0], %1;" ::"l"(tab + slot), "h"((uint16_t)v) : "memory");
#else
        asm volatile("st.global.cg.L2::cache_hint.u16 [%0], %1, %2;" ::"l"(tab + slot), "h"((uint16_t)v), "l"(l2_keep_policy()) : "memory");
#endif
    } else tab[slot] = (uint16_t)v;
}
template <bool kGT>
__device__ __forceinline__ void tab_put(uint32_t *tab, uint32_t slot, uint32_t v)
{
    if constexpr (kGT)
        asm volatile("st.global.cg.L2::cache_hint.u32 [%0], %1, %2;" ::"l"(tab + slot), "r"(v), "l"(l2_keep_policy()) : "memory");
    else tab[slot] = v;
}
template <bool kGT>
__device__ __forceinline__ void tab_fill16(uint4 *at, uint32_t f)
{
    if constexpr (kGT)
        asm volatile("st.global.cg.L2::cache_hint.v4.u32 [%0], {%1, %1, %1, %1}, %2;" ::"l"(at), "r"(f), "l"(l2_keep_policy()) : "memory");
    else *at = make_uint4(f, f, f, f);
}

// kTag (global u32 tables, blocks <= 64 KiB): an entry is (tag << 16) | position, tag = 16 bits hashed from the 4 bytes
// at that position.  A probe fetches its candidate's bytes only when the tags agree — a tag mismatch proves the 4-byte
// comparison of compress.rs:432-438 fails, so the parse is unchanged — which removes ~30 of the 32 speculative sector
// reads of a batch (most of the DRAM traffic of the untagged kernel).
__device__ __forceinline__ uint32_t tag16(uint32_t v4) { return (v4 * 2246822519u) >> 16; }

template <typename TabT, bool kGT = false, bool kTag = false, typename View = WordView>
__device__ __forceinline__ void match_block_view(View &view, uint32_t n, TabT *tab, uint32_t *ring,
                                                 bool cont, bool h5, SeqProducer &pr, uint32_t lane)
{
    static_assert(!kTag || (kGT && sizeof(TabT) == 4), "tagged entries: global u32 tables");
    constexpr uint32_t kInvalid = kTag ? 0xffffffffu : TabTraits<TabT>::kInvalid;
    const uint32_t lt_mask = (1u << lane) - 1u;
#ifdef LZ4B200_ENC_PROFILE
    EncProfile prof;
#endif
    ENC_PROF(start());
    if (n < 13) {                                               // compress.rs:343-346
        pr.push_final(0, n, lane);
        ENC_PROF(flush(lane));
        return;
    }
    view.advance(0u);
    {
        constexpr uint32_t words = 4096 * sizeof(TabT) / 16;
        uint32_t f = cont ? 0xffffffffu : 0u;
        if (kTag && !cont) {                                    // an empty slot is a candidate at position 0 (compress.rs:353-359):
            uint32_t lo0, hi0; view.ro5(0, lo0, hi0);           // it must carry position 0's real tag
            f = tag16(lo0) << 16;
        }
        uint4 *t128 = reinterpret_cast<uint4 *>(tab);
#pragma unroll 4
        for (uint32_t i = lane; i < words; i += 32) tab_fill16<kGT>(t128 + i, f);
        __syncwarp();
    }
    InputWindow win;
#if ENC_WINDOW
    win.init(reinterpret_cast<const uint8_t *>(view.w) + view.mis, n, ring);
#endif
    const uint32_t last_probe = n - 12;
    const uint32_t lim = n - 6;                                 // matches end before the last END_OFFSET bytes
    uint32_t anchor = 0, cur = 0;
    bool ri = false;                                            // T[H(cur-2)] = cur-2 still owed (compress.rs:460-461)
    if (!cont) {                                                // compress.rs:353-359
        uint32_t lo, hi; view.ro5(0, lo, hi);
        const uint32_t s = h5 ? slot_h5(lo, hi) : slot_h4(lo);
        if (lane == 0) tab_put<kGT>(tab, s, kTag ? tag16(lo) << 16 : 0u);
        cur = 1;
        __syncwarp();
    }
    ENC_PROF(phase(kPhSetup));

    for (;;) {                                                  // one sequence per iteration
#if ENC_WINDOW
        win.advance(cur + win.mis, lane);
#endif
        // ENC_FIRST_WIDTH < 32 (A/B aid): the first 32 probes (step 1) go in two rounds of ENC_FIRST_WIDTH and
        // 32 - ENC_FIRST_WIDTH lanes, trading speculative table/candidate traffic for an extra round on long searches.
        uint32_t base = cur, stride = 1, width = ENC_FIRST_WIDTH, cand, mpos;
        bool in_win = ENC_WINDOW != 0;                          // first batch: probe bytes come from the ring
        for (;;) {                                              // probe batches: compress.rs:373-439
            ENC_PROF(count(kCtBatch));
            view.advance(base);
            const uint32_t p = base + lane * stride;
            const bool act = lane < width;
            const bool term = act && p > last_probe;
            const bool live = act && !term;
            uint32_t v4, hi;
            if (in_win) win.ro5(p + win.mis, v4, hi);           // term lanes read ring bytes they never use
            else view.ro5(live ? p : 0u, v4, hi);
            uint32_t s2 = 0xffffffffu;
            if (ri) {
                // The re-insert of the previous sequence (compress.rs:460-461) rides along with the first probe loads.
                uint32_t lo2, hi2;
                if (ENC_WINDOW) win.ro5(cur - 2u + win.mis, lo2, hi2); else view.ro5(cur - 2u, lo2, hi2);
                s2 = h5 ? slot_h5(lo2, hi2) : slot_h4(lo2);
#if !ENC_RI_PATCH
                if (lane == 0) tab_put<kGT>(tab, s2, kTag ? ((cur - 2u) | (tag16(lo2) << 16)) : cur - 2u);
                __syncwarp();
                s2 = 0xffffffffu;
#endif
                ri = false;
            }
            uint32_t key = h5 ? slot_h5(v4, hi) : slot_h4(v4);
            uint32_t cnd = kInvalid;
            if (live) cnd = tab_get<kGT>(tab, key); else key = 0x10000u | lane;
            const uint32_t mytag = kTag ? tag16(v4) : 0u;
            bool tag_ok = true;
            if (kTag) { tag_ok = cnd != kInvalid && (cnd >> 16) == mytag; if (cnd != kInvalid) cnd &= 0xffffu; }
#if ENC_RI_PATCH
            // Nothing waits for the re-insert's table write: a probe on the same slot takes cur-2 directly and the
            // write itself is made with this batch's commits (dropped if a committed probe overwrites the slot).
            if (key == s2) cnd = cur - 2u;
#endif
            // The sequential loop overwrites T[h] before the next probe, so a probe sees the write of an earlier probe
            // of this batch when their slots collide.  First check the table's pre-batch candidates speculatively:
            // if none of the probes up to the first speculative hit w0 shares its slot with an earlier probe, the
            // speculation was exact.  For w0 <= 3 (89 % of JSON sequences) that is settled with three shuffles;
            // match.any — whose latency grows with the number of distinct keys, ~900 cycles for 32 — only runs
            // for the rest.
            bool chk = live && cnd != kInvalid && p - cnd <= 65535u && tag_ok;
            bool hit;
            if (kTag) {                                         // only lanes whose tag agrees touch memory
                uint32_t c4 = ~v4;
                if (chk) c4 = view.ro4(cnd);
                hit = chk & (c4 == v4);
            } else {
                hit = chk & (view.ro4(chk ? cnd : 0u) == v4);
            }
            uint32_t hits = __ballot_sync(kFull, hit);
            const uint32_t terms = (base + 31u * stride > last_probe) ? __ballot_sync(kFull, term) : 0u;   // uniform: only near the block's end
            ENC_PROF(phase(kPhProbe));
            const uint32_t w0 = hits ? (uint32_t)__ffs(hits) - 1u : 32u;
            uint32_t same = 1u << lane;                         // lanes of this batch on my slot (incl. me)
            bool exact = w0 == 0u;
#if ENC_FASTW
            if (w0 >= 1u && w0 <= 3u) {
                const uint32_t k0 = __shfl_sync(kFull, key, 0), k1 = __shfl_sync(kFull, key, 1), k2 = __shfl_sync(kFull, key, 2);
                const bool clash = (lane >= 1u && key == k0) || (lane >= 2u && key == k1) || (lane >= 3u && key == k2);
                exact = (__ballot_sync(kFull, clash && lane <= w0) == 0u);
            }
#endif
            if (!exact) {
                same = __match_any_sync(kFull, key);
                const uint32_t prior = same & lt_mask;
                const uint32_t le0 = w0 >= 31u ? kFull : ((2u << w0) - 1u);
                if (__ballot_sync(kFull, prior != 0u) & le0) {
                    if (kTag) {                                              // the forwarded candidate is a probe of this batch:
                        const uint32_t pl = prior ? 31u - __clz(prior) : lane;   // its 4 bytes sit in that lane's register
                        const uint32_t pv = __shfl_sync(kFull, v4, pl);
                        if (prior) { cnd = base + pl * stride; hit = pv == v4; }
                    } else if (prior) {
                        cnd = base + (31u - __clz(prior)) * stride;          // forwarded in-batch write
                        chk = p - cnd <= 65535u;                             // lanes with a prior are never term lanes
                        hit = chk & (view.ro4(chk ? cnd : 0u) == v4);
                    }
                    hits = __ballot_sync(kFull, hit);
                }
            }
            ENC_PROF(phase(kPhResolve));
            const uint32_t win = hits ? (uint32_t)__ffs(hits) - 1u : 32u;
            const uint32_t tfirst = terms ? (uint32_t)__ffs(terms) - 1u : 32u;
            if (tfirst < win) {                                 // compress.rs:381-384: the rest is literals
                pr.push_final(anchor, n, lane);
                ENC_PROF(phase(kPhPush));
                ENC_PROF(flush(lane));
                return;
            }
            // commit the table writes of probes 0..win (last writer per slot wins)
            const uint32_t upto = win < 32u ? win : width - 1u;
            const uint32_t le_mask = upto == 31u ? kFull : ((2u << upto) - 1u);
            const uint32_t mine = same & le_mask;
            if (lane <= upto && (31u - __clz(mine)) == lane) tab_put<kGT>(tab, key, kTag ? (p | (mytag << 16)) : p);
#if ENC_RI_PATCH
            if (s2 != 0xffffffffu) {                            // uniform: first batch after a match
                const uint32_t dups = __ballot_sync(kFull, key == s2 && lane <= upto);
                if (lane == 0 && dups == 0u) tab_put<kGT>(tab, s2, cur - 2u);
            }
#endif
            __syncwarp();
            ENC_PROF(phase(kPhCommit));
            if (win < 32u) {
                mpos = base + win * stride;
                cand = __shfl_sync(kFull, cnd, win);
                break;
            }
            base += width * stride;
            if (ENC_FIRST_WIDTH < 32 && base == cur + ENC_FIRST_WIDTH) {
                width = 32u - ENC_FIRST_WIDTH;                  // the rest of the step-1 probes
            } else {
                width = 32u;
                stride++;
            }
            in_win = false;
        }
        const uint32_t dist = mpos - cand;

        // ---- extension: the first forward round (32 bytes) and the backward round share one memory round trip
        const uint32_t room = min(cand, mpos - anchor);         // how far both sides may step back (0 for literal-free sequences)
        const uint32_t qf = mpos + 4u + lane;
        const bool inf = qf < lim;
        const uint8_t f1 = in_win ? win.byte(qf + win.mis) : view.byte(inf ? qf : mpos);
        const uint8_t f2 = view.byte((inf ? qf : mpos) - dist);
        uint32_t kb = 0;
        if (room) {                                             // compress.rs:272-287
            const bool inb = lane < room;
            const uint8_t b1 = view.byte(mpos - (inb ? 1u + lane : 0u)), b2 = view.byte(cand - (inb ? 1u + lane : 0u));
            const uint32_t bad = ~__ballot_sync(kFull, inb && b1 == b2);
            kb = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
        }
        const uint32_t badf = ~__ballot_sync(kFull, inf && f1 == f2);
        const uint32_t kf = badf ? (uint32_t)__ffs(badf) - 1u : 32u;
        uint32_t end = mpos + 4u + kf;
        if (kb) {
            mpos -= kb; cand -= kb;
            while (kb == 32u) {                                 // more than 32 bytes backwards: rare
                const uint32_t room2 = min(cand, mpos - anchor);
                const bool inb = lane < room2;
                const uint8_t b1 = view.byte(mpos - (inb ? 1u + lane : 0u)), b2 = view.byte(cand - (inb ? 1u + lane : 0u));
                const uint32_t bad = ~__ballot_sync(kFull, inb && b1 == b2);
                kb = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
                mpos -= kb; cand -= kb;
            }
        }
        if (kf == 32u) {                                        // long match: 128 bytes per round (compress.rs:156-216)
            for (;;) {
                view.advance(end);
                const uint32_t pos = end + 4u * lane;
                const bool full = pos + 4u <= lim;              // this lane's word lies before n - END_OFFSET
                const uint32_t x = view.ro4(full ? pos : 0u) ^ view.ro4(full ? pos - dist : 0u);
                const uint32_t nm = full ? (x ? (uint32_t)(__ffs(x) - 1) >> 3 : 4u) : 0u;
                const uint32_t bad = __ballot_sync(kFull, nm < 4u);
                if (bad) {
                    const uint32_t fl = (uint32_t)__ffs(bad) - 1u;
                    end += 4u * fl + __shfl_sync(kFull, nm, fl);
                    break;
                }
                end += 128u;
            }
            if (end < lim) {                                    // a word that crossed n - 6: at most 3 more bytes
                const uint32_t q = end + lane;
                const bool ok = lane < 4u && q < lim && view.byte(q < lim ? q : end) == view.byte((q < lim ? q : end) - dist);
                end += (uint32_t)__ffs(~__ballot_sync(kFull, ok)) - 1u;
            }
        }
        ENC_PROF(phase(kPhExtend));
        ENC_PROF(count(kCtSeq));
        ENC_PROF(count(kCtNoBack, room == 0u));
        ENC_PROF(count(kCtShort, room == 0u && kf < 8u));
        ENC_PROF(count(kCtLong, kf == 32u));
        pr.push(anchor, mpos, dist, end, lane);
        ENC_PROF(phase(kPhPush));
        anchor = cur = end;
        ri = true;
    }
}

template <typename TabT, bool kGT = false, bool kTag = false>
__device__ __forceinline__ void match_block(const uint8_t *__restrict__ src, uint32_t n, TabT *tab, uint32_t *ring,
                                            bool cont, bool h5, SeqProducer &pr, uint32_t lane)
{
    WordView view(src);
    match_block_view<TabT, kGT, kTag>(view, n, tab, ring, cont, h5, pr, lane);
}

#ifdef LZ4B200_AB_VARIANTS   // measured and rejected (DESIGN.md §6): A/B build only
// ---------------------------------------------------------------------------------------------
// Matcher with 4-bit tags in SHARED memory beside the global position table (lz4_compress_blocks_gnib).
// What `gtab` pays for its 56 chains per SM is table and candidate traffic: every probe batch loads 32 table entries
// and 32 candidates although the sequential loop of compress.rs:373-439 stops at the first match, 2.4 probes in on JSON.  Here every
// slot also has a 4-bit tag of the 4 bytes at its position, 2 KiB per chain in shared memory (8 x 7 chains = 112 KB per
// SM).  A probe whose tag disagrees cannot pass the 4-byte comparison (compress.rs:432-438), so it touches neither the
// table nor its candidate.  The tag-matching probes are verified TWO at a time in probe order and the search stops at
// the first real hit — exactly the probes the sequential loop would have executed, plus at most one.  Exactness of the
// in-batch forwarding is kept as in match_block: clashes among the probes up to the hit are detected (three shuffles /
// match.any) and re-evaluated register to register; if that takes the hit away and nothing before it matches, the probes
// up to there are committed and the batch continues behind them inside the same 32-probe step group (`gi`).
// Model + proof against the oracle: tests/test_warp_emulation.py::warp_encode_nib.
// ---------------------------------------------------------------------------------------------
// Tag storage: kTagBits = 4 -> nibbles, 2 KiB per chain, updated with two shared-memory reductions (lanes of one commit
// may own different nibbles of a word); kTagBits = 8 -> bytes, 4 KiB per chain, plain byte stores.  The chain's tag array
// and its table are addressed through two opaque 32-bit values (a shared-memory address and a byte offset from the table
// base): with 32-40 registers per thread the compiler otherwise re-derives both pointers from threadIdx / blockIdx in
// every divergent block (~30 instructions each).
template <int kTagBits> __device__ __forceinline__ uint32_t tagof(uint32_t v4) { return (v4 * 2246822519u) >> (32 - kTagBits); }

__device__ __forceinline__ uint32_t opaque32(uint32_t v) { asm volatile("mov.b32 %0, %0;" : "+r"(v)); return v; }

template <int kTagBits>
__device__ __forceinline__ uint32_t tag_get(uint32_t nt_sa, uint32_t slot)
{
    uint32_t v;
    if constexpr (kTagBits == 8) {
        asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(nt_sa + slot) : "memory");
        return v;
    } else {                                                     // 4- or 2-bit tags packed into 32-bit words
        const uint32_t bit = slot * kTagBits;
        asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(nt_sa + ((bit >> 3) & ~3u)) : "memory");
        return (v >> (bit & 31u)) & ((1u << kTagBits) - 1u);
    }
}
template <int kTagBits>
__device__ __forceinline__ void tag_put(uint32_t nt_sa, uint32_t slot, uint32_t tag)
{
    if constexpr (kTagBits == 8) {
        asm volatile("st.shared.u8 [%0], %1;" ::"r"(nt_sa + slot), "r"(tag) : "memory");
    } else {
        const uint32_t bit = slot * kTagBits, sa = nt_sa + ((bit >> 3) & ~3u), sh = bit & 31u;
        asm volatile("red.shared.and.b32 [%0], %1;" ::"r"(sa), "r"(~(((1u << kTagBits) - 1u) << sh)) : "memory");
        asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(sa), "r"(tag << sh) : "memory");
    }
}
template <int kTagBits> __device__ __forceinline__ uint32_t tag_fill_word(uint32_t t)
{
    return kTagBits == 8 ? t * 0x01010101u : kTagBits == 4 ? t * 0x11111111u : t * 0x55555555u;
}
__device__ __forceinline__ uint32_t gpos_get(const uint8_t *gtab, uint32_t tab_off, uint32_t slot)
{
    uint16_t v;
    asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(v) : "l"(gtab + (tab_off + slot * 2u)) : "memory");
    return v;
}
__device__ __forceinline__ void gpos_put(uint8_t *gtab, uint32_t tab_off, uint32_t slot, uint32_t pos)
{
    asm volatile("st.global.cg.u16 [%0], %1;" ::"l"(gtab + (tab_off + slot * 2u)), "h"((uint16_t)pos) : "memory");
}

template <int kTagBits, typename View>
__device__ __forceinline__ void match_block_nib(View &view, uint32_t n, uint8_t *gtab, uint32_t tab_off, uint32_t nt_sa,
                                                bool cont, bool h5, SeqProducer &pr, uint32_t lane)
{
    constexpr uint32_t kInvalid = TabTraits<uint16_t>::kInvalid;
    const uint32_t lt_mask = (1u << lane) - 1u;
    if (n < 13) {                                               // compress.rs:343-346
        pr.push_final(0, n, lane);
        return;
    }
    view.advance(0u);
    {
        const uint32_t f = cont ? 0xffffffffu : 0u;
        uint4 *t128 = reinterpret_cast<uint4 *>(gtab + tab_off);
#pragma unroll 4
        for (uint32_t i = lane; i < 4096u * 2u / 16u; i += 32)
            asm volatile("st.global.cg.v4.u32 [%0], {%1, %1, %1, %1};" ::"l"(t128 + i), "r"(f) : "memory");
        uint32_t lo0, hi0; view.ro5(0, lo0, hi0);               // an empty slot is a candidate at position 0: its tag
        const uint32_t t = tag_fill_word<kTagBits>(tagof<kTagBits>(lo0));
#pragma unroll
        for (uint32_t i = lane; i < 4096u * kTagBits / 8u / 16u; i += 32)
            asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(nt_sa + i * 16u), "r"(t) : "memory");
        __syncwarp();
    }
    const uint32_t last_probe = n - 12;
    const uint32_t lim = n - 6;
    uint32_t anchor = 0, cur = 0;
    bool ri = false;
    if (!cont) {                                                // compress.rs:353-359
        uint32_t lo, hi; view.ro5(0, lo, hi);
        const uint32_t s = h5 ? slot_h5(lo, hi) : slot_h4(lo);
        if (lane == 0) { gpos_put(gtab, tab_off, s, 0u); tag_put<kTagBits>(nt_sa, s, tagof<kTagBits>(lo)); }
        cur = 1;
        __syncwarp();
    }

    for (;;) {                                                  // one sequence per iteration
        uint32_t gbase = cur, stride = 1, gi = 0, cand, mpos;
        for (;;) {                                              // probe batches: compress.rs:373-439
            const uint32_t width = 32u - gi;
            const uint32_t base = gbase + gi * stride;
            view.advance(base);
            const uint32_t p = base + lane * stride;
            const bool act = lane < width;
            const bool term = act && p > last_probe;
            const bool live = act && !term;
            uint32_t v4, hi;
            view.ro5(live ? p : 0u, v4, hi);
            if (ri) {                                           // compress.rs:460-461, before this batch's table reads
                uint32_t lo2, hi2;
                view.ro5(cur - 2u, lo2, hi2);
                const uint32_t s2 = h5 ? slot_h5(lo2, hi2) : slot_h4(lo2);
                if (lane == 0) { gpos_put(gtab, tab_off, s2, cur - 2u); tag_put<kTagBits>(nt_sa, s2, tagof<kTagBits>(lo2)); }
                __syncwarp();
                ri = false;
            }
            uint32_t key = h5 ? slot_h5(v4, hi) : slot_h4(v4);
            const uint32_t mytag = tagof<kTagBits>(v4);
            bool tm = false;
            if (live) tm = tag_get<kTagBits>(nt_sa, key) == mytag; else key = 0x10000u | lane;
            uint32_t pend = __ballot_sync(kFull, tm);
            uint32_t cnd = kInvalid, hits = 0;
            bool hit = false;
            while (pend) {                                      // verify the tag-matching probes two at a time, in order
                const uint32_t rest = pend & (pend - 1u), rest2 = rest & (rest - 1u);
                const bool sel = ((pend & ~rest2) >> lane) & 1u;
                if (sel) {
                    cnd = gpos_get(gtab, tab_off, key);
                    const bool chk = cnd != kInvalid && p - cnd <= 65535u;
                    hit = chk && view.ro4(chk ? cnd : 0u) == v4;
                }
                hits = __ballot_sync(kFull, sel && hit);
                if (hits) break;
                pend = rest2;
            }
            const uint32_t terms = (gbase + 31u * stride > last_probe) ? __ballot_sync(kFull, term) : 0u;
            const uint32_t w0 = hits ? (uint32_t)__ffs(hits) - 1u : 32u;
            const uint32_t upto0 = w0 < width ? w0 : width - 1u;
            uint32_t same = 1u << lane, win = w0;
            bool exact = w0 == 0u;
            if (w0 >= 1u && w0 <= 3u) {
                const uint32_t k0 = __shfl_sync(kFull, key, 0), k1 = __shfl_sync(kFull, key, 1), k2 = __shfl_sync(kFull, key, 2);
                const bool clash = (lane >= 1u && key == k0) || (lane >= 2u && key == k1) || (lane >= 3u && key == k2);
                exact = (__ballot_sync(kFull, clash && lane <= w0) == 0u);
            }
            if (!exact) {
                same = __match_any_sync(kFull, key);
                const uint32_t prior = same & lt_mask;
                const uint32_t le0 = upto0 >= 31u ? kFull : ((2u << upto0) - 1u);
                if (__ballot_sync(kFull, prior != 0u) & le0) {
                    const uint32_t pl = prior ? 31u - __clz(prior) : lane;   // the forwarded candidate is a probe of this
                    const uint32_t pv = __shfl_sync(kFull, v4, pl);          // batch: its 4 bytes sit in that lane's register
                    if (prior) { cnd = base + pl * stride; hit = pv == v4; }
                    const uint32_t h2 = __ballot_sync(kFull, hit) & le0;
                    win = h2 ? (uint32_t)__ffs(h2) - 1u : 32u;
                }
            }
            const bool partial = win == 32u && w0 < 32u;        // forwarding took the hit away: probes 0..w0 were executed
            const uint32_t tfirst = terms ? (uint32_t)__ffs(terms) - 1u : 32u;
            if (!partial && tfirst < win) {                     // compress.rs:381-384: the rest is literals
                pr.push_final(anchor, n, lane);
                return;
            }
            const uint32_t upto = partial ? w0 : (win < 32u ? win : width - 1u);
            const uint32_t le_mask = upto == 31u ? kFull : ((2u << upto) - 1u);
            const uint32_t mine = same & le_mask;
            if (lane <= upto && (31u - __clz(mine)) == lane) { gpos_put(gtab, tab_off, key, p); tag_put<kTagBits>(nt_sa, key, mytag); }
            __syncwarp();
            if (win < 32u) {
                mpos = base + win * stride;
                cand = __shfl_sync(kFull, cnd, win);
                break;
            }
            gi += upto + 1u;
            if (gi == 32u) { gbase += 32u * stride; stride++; gi = 0; }
        }
        const uint32_t dist = mpos - cand;

        // ---- extension (as match_block_view): first forward round and the backward round share one round trip
        const uint32_t room = min(cand, mpos - anchor);
        const uint32_t qf = mpos + 4u + lane;
        const bool inf = qf < lim;
        const uint8_t f1 = view.byte(inf ? qf : mpos);
        const uint8_t f2 = view.byte((inf ? qf : mpos) - dist);
        uint32_t kb = 0;
        if (room) {                                             // compress.rs:272-287
            const bool inb = lane < room;
            const uint8_t b1 = view.byte(mpos - (inb ? 1u + lane : 0u)), b2 = view.byte(cand - (inb ? 1u + lane : 0u));
            const uint32_t bad = ~__ballot_sync(kFull, inb && b1 == b2);
            kb = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
        }
        const uint32_t badf = ~__ballot_sync(kFull, inf && f1 == f2);
        const uint32_t kf = badf ? (uint32_t)__ffs(badf) - 1u : 32u;
        uint32_t end = mpos + 4u + kf;
        if (kb) {
            mpos -= kb; cand -= kb;
            while (kb == 32u) {
                const uint32_t room2 = min(cand, mpos - anchor);
                const bool inb = lane < room2;
                const uint8_t b1 = view.byte(mpos - (inb ? 1u + lane : 0u)), b2 = view.byte(cand - (inb ? 1u + lane : 0u));
                const uint32_t bad = ~__ballot_sync(kFull, inb && b1 == b2);
                kb = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
                mpos -= kb; cand -= kb;
            }
        }
        if (kf == 32u) {                                        // long match: 128 bytes per round (compress.rs:156-216)
            for (;;) {
                view.advance(end);
                const uint32_t pos = end + 4u * lane;
                const bool full = pos + 4u <= lim;
                const uint32_t x = view.ro4(full ? pos : 0u) ^ view.ro4(full ? pos - dist : 0u);
                const uint32_t nm = full ? (x ? (uint32_t)(__ffs(x) - 1) >> 3 : 4u) : 0u;
                const uint32_t bad = __ballot_sync(kFull, nm < 4u);
                if (bad) {
                    const uint32_t fl = (uint32_t)__ffs(bad) - 1u;
                    end += 4u * fl + __shfl_sync(kFull, nm, fl);
                    break;
                }
                end += 128u;
            }
            if (end < lim) {
                const uint32_t q = end + lane;
                const bool ok = lane < 4u && q < lim && view.byte(q < lim ? q : end) == view.byte((q < lim ? q : end) - dist);
                end += (uint32_t)__ffs(~__ballot_sync(kFull, ok)) - 1u;
            }
        }
        pr.push(anchor, mpos, dist, end, lane);
        anchor = cur = end;
        ri = true;
    }
}

#endif  // LZ4B200_AB_VARIANTS (shared-memory tag matcher)

// ---------------------------------------------------------------------------------------------
// matcher with an external dictionary: compress_into_with_dict (compress.rs:554-583, 610-616).
// The dictionary logically precedes the input: the table holds STREAM positions (input position + dictionary
// length), init_dict seeds it with every third dictionary position, and a candidate below the dictionary
// length is matched against the dictionary's bytes (compress.rs:412-421) — backwards to its first byte,
// forwards to its last (a match never runs from the dictionary into the input).  This path is about
// completeness, not speed: plain global loads, full match.any per batch.
// ---------------------------------------------------------------------------------------------
template <typename TabT>
__device__ __forceinline__ void match_block_dict(const uint8_t *__restrict__ src, uint32_t n,
                                                 const uint8_t *__restrict__ dict, uint32_t dlen, TabT *tab, bool h5,
                                                 SeqProducer &pr, uint32_t lane)
{
    const uint32_t lt_mask = (1u << lane) - 1u;
    const uint32_t off = dlen;                                  // input_stream_offset
    if (n < 13) {                                               // compress.rs:343-346
        pr.push_final(0, n, lane);
        return;
    }
    {
        constexpr uint32_t words = 4096 * sizeof(TabT) / 16;
        uint4 *t128 = reinterpret_cast<uint4 *>(tab);
        for (uint32_t i = lane; i < words; i += 32) t128[i] = make_uint4(0u, 0u, 0u, 0u);
        __syncwarp();
    }
    const WordView view(src), dview(dict);
    // init_dict (compress.rs:571-583): positions 0, 3, 6, ... with 8 readable bytes, in order; the last writer of
    // a slot wins, within a batch of 32 that is the highest lane
    for (uint32_t i0 = 0; i0 + 8u <= dlen; i0 += 96u) {
        const uint32_t i = i0 + 3u * lane;
        const bool act = i + 8u <= dlen;
        uint32_t lo, hi; dview.ro5(act ? i : 0u, lo, hi);
        const uint32_t key = act ? (h5 ? slot_h5(lo, hi) : slot_h4(lo)) : (0x10000u | lane);
        const uint32_t same = __match_any_sync(kFull, key);
        if (act && (31u - __clz(same)) == lane) tab[key] = (TabT)i;
        __syncwarp();
    }
    const uint32_t last_probe = n - 12;
    const uint32_t lim = n - 6;
    uint32_t anchor = 0, cur = 0;
    bool ri = false;
    for (;;) {                                                  // one sequence per iteration
        uint32_t base = cur, stride = 1, cand_s, mpos;
        for (;;) {                                              // probe batches: compress.rs:373-439
            const uint32_t p = base + lane * stride;
            const bool term = p > last_probe;
            uint32_t v4, hi;
            view.ro5(term ? 0u : p, v4, hi);
            if (ri) {                                           // compress.rs:460-461
                uint32_t lo2, hi2; view.ro5(cur - 2u, lo2, hi2);
                const uint32_t s2 = h5 ? slot_h5(lo2, hi2) : slot_h4(lo2);
                if (lane == 0) tab[s2] = (TabT)(cur - 2u + off);
                __syncwarp();
                ri = false;
            }
            uint32_t key = h5 ? slot_h5(v4, hi) : slot_h4(v4);
            uint32_t cnd = 0;                                   // stream position of the candidate
            if (!term) cnd = tab[key]; else key = 0x10000u | lane;
            const uint32_t same = __match_any_sync(kFull, key);
            const uint32_t prior = same & lt_mask;
            if (prior) cnd = off + base + (31u - __clz(prior)) * stride;   // forwarded in-batch write
            const bool chk = !term && p + off - cnd <= 65535u;
            const bool in_dict = cnd < off;
            const uint32_t c4 = in_dict ? dview.ro4s(chk ? cnd : 0u) : view.ro4(chk ? cnd - off : 0u);
            const bool hit = chk & (c4 == v4);
            const uint32_t hits = __ballot_sync(kFull, hit), terms = __ballot_sync(kFull, term);
            const uint32_t win = hits ? (uint32_t)__ffs(hits) - 1u : 32u;
            const uint32_t tfirst = terms ? (uint32_t)__ffs(terms) - 1u : 32u;
            if (tfirst < win) {                                 // compress.rs:381-384
                pr.push_final(anchor, n, lane);
                return;
            }
            const uint32_t upto = win < 32u ? win : 31u;
            const uint32_t le_mask = upto == 31u ? kFull : ((2u << upto) - 1u);
            const uint32_t mine = same & le_mask;
            if (lane <= upto && (31u - __clz(mine)) == lane) tab[key] = (TabT)(p + off);
            __syncwarp();
            if (win < 32u) {
                mpos = base + win * stride;
                cand_s = __shfl_sync(kFull, cnd, win);
                break;
            }
            base += 32u * stride;
            stride++;
        }
        const uint32_t dist = mpos + off - cand_s;
        const bool cd = cand_s < off;                           // candidate lives in the dictionary
        const uint8_t *__restrict__ cs = cd ? dict : src;
        const uint32_t clen = cd ? dlen : n;
        uint32_t ci = cd ? cand_s : cand_s - off;               // its index in its own buffer
        for (;;) {                                              // backwards: compress.rs:272-287
            const uint32_t room = min(ci, mpos - anchor);
            const bool ok = lane < room && __ldg(src + mpos - (lane < room ? 1u + lane : 0u)) == __ldg(cs + ci - (lane < room ? 1u + lane : 0u));
            const uint32_t bad = ~__ballot_sync(kFull, ok);
            const uint32_t kb = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
            mpos -= kb; ci -= kb;
            if (kb < 32u) break;
        }
        uint32_t end = mpos + 4u, cj = ci + 4u;
        for (;;) {                                              // forwards: compress.rs:156-216 (input and source limits)
            const uint32_t q = end + lane, cq = cj + lane;
            const bool in = q < lim && cq < clen;
            const bool ok = in && __ldg(src + (in ? q : mpos)) == __ldg(cs + (in ? cq : ci));
            const uint32_t bad = ~__ballot_sync(kFull, ok);
            const uint32_t k = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
            end += k; cj += k;
            if (k < 32u) break;
        }
        pr.push(anchor, mpos, dist, end, lane);
        anchor = cur = end;
        ri = true;
    }
}

// ---------------------------------------------------------------------------------------------
// emitter: compress.rs:463-486 for 32 sequences at a time.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint8_t *put_len_ext(uint8_t *p, uint32_t v)     // v = length - 15 (write_integer, compress.rs:217-242)
{
    while (v >= 255u) { *p++ = 0xff; v -= 255u; }
    *p++ = (uint8_t)v;
    return p;
}

// Emits one batch of tuples (one per lane) at output cursor `o`; returns the bytes produced.
__device__ __forceinline__ uint32_t emit_batch(const uint8_t *__restrict__ src, uint8_t *dst, uint32_t o, const uint4 e,
                                               uint32_t cnt, uint32_t lane)
{
    const bool valid = lane < cnt;
    const bool tail = e.z == 0;                            // last literals: no match part
    const uint32_t lit = valid ? (tail ? e.w : e.y) - e.x : 0u;
    const uint32_t extra = (valid && !tail) ? e.w - e.y - 4u : 0u;
    const uint32_t lit_ext = lit >= 15u ? (lit - 15u) / 255u + 1u : 0u;
    const uint32_t m_ext = extra >= 15u ? (extra - 15u) / 255u + 1u : 0u;
    const uint32_t size = valid ? 1u + lit_ext + lit + (tail ? 0u : 2u + m_ext) : 0u;
    uint32_t incl = size;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(kFull, incl, d);
        if (lane >= (uint32_t)d) incl += t;
    }
    const uint32_t total = __shfl_sync(kFull, incl, 31);
    uint8_t *p = dst + o + (incl - size);
    uint8_t *lit_at = p;
    if (valid) {
        *p++ = (uint8_t)(((lit < 15u ? lit : 15u) << 4) | (tail ? 0u : (extra < 15u ? extra : 15u)));
        if (lit >= 15u) p = put_len_ext(p, lit - 15u);
        lit_at = p;
        if (lit <= kSmallLit) {
            // 8 bytes per round trip (loads first, then stores): a byte-at-a-time loop pays one L2 latency per byte
            const uint8_t *s = src + e.x;
            for (uint32_t i = 0; i < lit; i += 8u) {
                uint8_t c[8];
#pragma unroll
                for (uint32_t k = 0; k < 8u; k++) c[k] = (i + k < lit) ? __ldg(s + i + k) : (uint8_t)0;
#pragma unroll
                for (uint32_t k = 0; k < 8u; k++) if (i + k < lit) p[i + k] = c[k];
            }
        }
        p += lit;
        if (!tail) {
            p[0] = (uint8_t)e.z; p[1] = (uint8_t)(e.z >> 8);
            p += 2;
            if (extra >= 15u) put_len_ext(p, extra - 15u);
        }
    }
    // long literal runs: the whole warp copies them, one run at a time
    uint32_t big = __ballot_sync(kFull, valid && lit > kSmallLit);
    while (big) {
        const uint32_t l = (uint32_t)__ffs(big) - 1u;
        big &= big - 1u;
        const uint32_t from = __shfl_sync(kFull, e.x, l), len = __shfl_sync(kFull, lit, l);
        const uint32_t at = __shfl_sync(kFull, (uint32_t)(lit_at - dst), l);
        const uint8_t *s = src + from;
        uint8_t *d = dst + at;
        uint32_t i = lane;
        for (; i + 96u < len; i += 128u) {
            const uint8_t c0 = __ldg(s + i), c1 = __ldg(s + i + 32), c2 = __ldg(s + i + 64), c3 = __ldg(s + i + 96);
            d[i] = c0; d[i + 32] = c1; d[i + 64] = c2; d[i + 96] = c3;
        }
        for (; i < len; i += 32u) d[i] = __ldg(s + i);
    }
    return total;
}

// Emitter serving one matcher (lz4_compress_blocks_split).
__device__ __forceinline__ void emit_loop(const BatchArgs &a, const uint4 *q, const volatile uint32_t *meta, uint64_t *bars,
                                          uint32_t lane)
{
    const uint8_t *src = nullptr;
    uint8_t *dst = nullptr;
    uint32_t o = 0;
    for (uint32_t j = 0;; j++) {
        const uint32_t h = j & 1u;
        mbar_wait_relaxed(bars + h, (j >> 1) & 1u);
        const uint32_t b = meta[h * 4 + 0], cnt = meta[h * 4 + 1], fl = meta[h * 4 + 2];
        uint4 e = make_uint4(0, 0, 0, 0);
        if (lane < cnt && b != kExitBlock) e = q[h * kSeqBatchEntries + lane];
        __syncwarp();
        if (lane == 0) mbar_arrive(bars + 2 + h);              // tuples are in registers: the half may be refilled
        if (b == kExitBlock) break;
        if (fl & 1u) { src = a.in + a.in_off[b]; dst = a.out + a.out_off[b]; o = 0; }
        o += emit_batch(src, dst, o, e, cnt, lane);
        if ((fl & 2u) && lane == 0) { a.out_len[b] = o; a.status[b] = LZ4B200_OK; }
    }
}

// Emitter serving kR matchers (lz4_compress_blocks_gtab): polls their rings in turn; per-ring state in shared memory.
struct EmitState { const uint8_t *src; uint8_t *dst; uint32_t o, j; };

template <int kR>
__device__ __forceinline__ void emit_loop_multi(const BatchArgs &a, const uint4 *q0, const volatile uint32_t *meta0,
                                                uint64_t *bars0, EmitState *st, uint32_t lane)
{
    if (lane < (uint32_t)kR) { st[lane].src = nullptr; st[lane].dst = nullptr; st[lane].o = 0; st[lane].j = 0; }
    __syncwarp();
    uint32_t live = (1u << kR) - 1u;
    while (live) {
        bool progress = false;
#pragma unroll 1
        for (int i = 0; i < kR; i++) {
            if (!((live >> i) & 1u)) continue;
            const uint4 *q = q0 + i * 2 * kSeqBatchEntries;
            const volatile uint32_t *meta = meta0 + i * 8;
            uint64_t *bars = bars0 + i * 4;
            const uint32_t j = st[i].j, h = j & 1u;
            uint32_t ready;
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.acquire.cta.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                         : "=r"(ready) : "r"(smem_addr(bars + h)), "r"((j >> 1) & 1u) : "memory");
            if (!ready) continue;
            progress = true;
            const uint32_t b = meta[h * 4 + 0], cnt = meta[h * 4 + 1], fl = meta[h * 4 + 2];
            uint4 e = make_uint4(0, 0, 0, 0);
            if (lane < cnt && b != kExitBlock) e = q[h * kSeqBatchEntries + lane];
            __syncwarp();
            if (lane == 0) { mbar_arrive(bars + 2 + h); st[i].j = j + 1u; }
            if (b == kExitBlock) { live &= ~(1u << i); __syncwarp(); continue; }
            if ((fl & 1u) && lane == 0) { st[i].src = a.in + a.in_off[b]; st[i].dst = a.out + a.out_off[b]; st[i].o = 0; }
            __syncwarp();
            const uint32_t o = st[i].o;
            const uint32_t total = emit_batch(st[i].src, st[i].dst, o, e, cnt, lane);
            __syncwarp();
            if (lane == 0) {
                st[i].o = o + total;
                if (fl & 2u) { a.out_len[b] = o + total; a.status[b] = LZ4B200_OK; }
            }
            __syncwarp();
        }
        if (!progress) __nanosleep(ENC_EMIT_SLEEP_NS ? ENC_EMIT_SLEEP_NS : 200);
    }
}

// One CTA = kPairs matcher warps (warps 0..kPairs-1) + kPairs emitter warps.  Shared memory per pair: the
// table (8 KiB for blocks <= 64 KiB, 16 KiB above), 512 bytes of tuples, the 512-byte input ring, 32 bytes of
// batch headers, 4 mbarriers.
template <typename TabT, int kPairs>
constexpr int split_ctas_per_sm()                              // what 227 KB of shared memory (1 KB reserved per CTA) holds
{
    return (int)((227u * 1024u) / (kPairs * (4096 * sizeof(TabT) + 2 * kSeqBatchEntries * 16 + kRingBytes + 64) + 1024u));
}

template <typename TabT, int kPairs, bool kDict>
__global__ void __launch_bounds__(kPairs * 64, split_ctas_per_sm<TabT, kPairs>())
lz4_compress_blocks_split(BatchArgs a, uint32_t *tickets)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t warp = threadIdx.x >> 5, lane = lane_id();
    const uint32_t pair = warp < (uint32_t)kPairs ? warp : warp - kPairs;
    TabT *tab = reinterpret_cast<TabT *>(smem_raw) + pair * 4096;
    constexpr size_t kTab = 4096 * sizeof(TabT), kQ = 2 * kSeqBatchEntries * 16;
    uint4 *q = reinterpret_cast<uint4 *>(smem_raw + kPairs * kTab) + pair * 2 * kSeqBatchEntries;
    uint32_t *ring = reinterpret_cast<uint32_t *>(smem_raw + kPairs * (kTab + kQ)) + pair * (kRingBytes / 4);
    uint32_t *meta = reinterpret_cast<uint32_t *>(smem_raw + kPairs * (kTab + kQ + kRingBytes)) + pair * 8;
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + kPairs * (kTab + kQ + kRingBytes + 32)) + pair * 4;
    if (threadIdx.x < (uint32_t)kPairs * 4u)
        mbar_init(reinterpret_cast<uint64_t *>(smem_raw + kPairs * (kTab + kQ + kRingBytes + 32)) + threadIdx.x, 1u);
    __syncthreads();
    if (warp >= (uint32_t)kPairs) {
        emit_loop(a, q, meta, bars, lane);
        return;
    }
    constexpr bool kSmall = sizeof(TabT) == 2;
    SeqProducer pr{q, meta, bars, 0u, 0u, 0u, 0u};
    for (uint32_t b = next_ticket(tickets); b < a.nblocks; b = next_ticket(tickets)) {
        const uint32_t n = a.in_len[b];
        const uint64_t span = (uint64_t)n + (kDict ? a.dict_len : 0u);      // table layout follows dict + input: compress.rs:559
        if ((span <= 65536u) != kSmall) continue;
        const uint32_t fl = a.flags ? a.flags[b] : 0u;
        if ((uint64_t)a.out_cap[b] < max_output_size_dev(n)) {              // compress.rs:338-340
            if (lane == 0) { a.out_len[b] = 0; a.status[b] = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL; }
            continue;
        }
        const bool h5 = (fl & LZ4B200_BLOCK_HASH5_ALWAYS) || span >= 65535u;
        pr.block = b; pr.first = 1;
        if constexpr (kDict)
            match_block_dict<TabT>(a.in + a.in_off[b], n, a.dict, a.dict_len, tab, h5, pr, lane);
        else
            match_block<TabT>(a.in + a.in_off[b], n, tab, ring, (fl & LZ4B200_BLOCK_CONT) != 0, h5, pr, lane);
    }
    pr.block = kExitBlock; pr.first = 0;
    pr.flush(0, lane);
    retire_warp(tickets, gridDim.x * kPairs);
}

// The per-warp block loop of a matcher (shared by the kernels below).
template <typename TabT, bool kGT, bool kTag = false>
__device__ __forceinline__ void matcher_loop(const BatchArgs &a, uint32_t *tickets, TabT *tab, SeqProducer &pr, uint32_t lane)
{
    constexpr bool kSmall = sizeof(TabT) == 2 || kTag;
    for (uint32_t b = next_ticket(tickets); b < a.nblocks; b = next_ticket(tickets)) {
        const uint32_t n = a.in_len[b];
        if ((n <= 65536u) != kSmall) continue;
        const uint32_t fl = a.flags ? a.flags[b] : 0u;
        if ((uint64_t)a.out_cap[b] < max_output_size_dev(n)) {              // compress.rs:338-340
            if (lane == 0) { a.out_len[b] = 0; a.status[b] = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL; }
            continue;
        }
        const bool h5 = (fl & LZ4B200_BLOCK_HASH5_ALWAYS) || n >= 65535u;
        pr.block = b; pr.first = 1;
        match_block<TabT, kGT, kTag>(a.in + a.in_off[b], n, tab, nullptr, (fl & LZ4B200_BLOCK_CONT) != 0, h5, pr, lane);
    }
    pr.block = kExitBlock; pr.first = 0;
    pr.flush(0, lane);
}

// Many-matcher variant: kM matcher warps + kE emitter warps per CTA (kM a multiple of kE).  The first kS matchers
// of a CTA keep their table in shared memory (kS x 8 KiB of dynamic shared memory); the other kM - kS keep it in global
// memory (gtab, 4096 entries for each of them, CTA after CTA).  Shared-memory tables cap an SM at 24 matchers; global tables cost
// ~250 cycles per access but none of the 228 KB.  Blocks are pulled from one ticket queue, so the faster
// shared-memory matchers simply take more of them.  kCtas: resident CTAs per SM the launch plans for (sets the
// register budget); the default fills all 64 warp slots.
template <typename TabT, int kM, int kE, int kS, int kCtas = 2048 / ((kM + kE) * 32)>
__global__ void __launch_bounds__((kM + kE) * 32, kCtas)
lz4_compress_blocks_gtab(BatchArgs a, uint32_t *tickets, TabT *gtab)
{
    constexpr int kR = kM / kE;
    static_assert(kM % kE == 0, "every emitter serves the same number of matchers");
    extern __shared__ __align__(16) uint8_t smem_raw[];      // kS tables
    __shared__ __align__(16) uint4 q_s[kM * 2 * kSeqBatchEntries];
    __shared__ uint32_t meta_s[kM * 8];
    __shared__ __align__(8) uint64_t bars_s[kM * 4];
    __shared__ EmitState st_s[kM];
    // The warp index comes from a warp reduction, which writes a uniform register: with threadIdx.x >> 5 the compiler cannot
    // tell that the role branches below are warp-uniform, and it then guards every shuffle, ballot and match.any of the
    // matcher and the emitter with a divergence check and a collective-emulation fall-back (88 of them in this kernel).
    const uint32_t warp = __reduce_max_sync(kFull, threadIdx.x >> 5), lane = lane_id();
    if (threadIdx.x < (uint32_t)kM * 4u) mbar_init(bars_s + threadIdx.x, 1u);
    __syncthreads();
    if (warp >= (uint32_t)kM) {
        const uint32_t e = warp - kM;
        emit_loop_multi<kR>(a, q_s + e * kR * 2 * kSeqBatchEntries, meta_s + e * kR * 8, bars_s + e * kR * 4,
                            st_s + e * kR, lane);
        return;
    }
    SeqProducer pr{q_s + warp * 2 * kSeqBatchEntries, meta_s + warp * 8, bars_s + warp * 4, 0u, 0u, 0u, 0u};
    if (kS > 0 && warp + 1u <= (uint32_t)kS)
        matcher_loop<TabT, false>(a, tickets, reinterpret_cast<TabT *>(smem_raw) + warp * 4096, pr, lane);
    else {
        // tables of the kM - kS global matchers only, CTA after CTA (the launcher reserves exactly that many)
#if ENC_TAB_OPAQUE
        uint32_t toff = (blockIdx.x * (kM - kS) + warp - kS) * 4096u;   // opaque: not re-derived from blockIdx / threadIdx at every use
        asm volatile("mov.b32 %0, %0;" : "+r"(toff));
        matcher_loop<TabT, true>(a, tickets, gtab + toff, pr, lane);
#else
        matcher_loop<TabT, true>(a, tickets, gtab + ((size_t)blockIdx.x * (kM - kS) + warp - kS) * 4096, pr, lane);
#endif
    }
    retire_warp(tickets, gridDim.x * kM);
}

#ifdef LZ4B200_AB_VARIANTS
// Global position tables + shared-memory tags (match_block_nib): kM matchers + kE emitters per CTA, kCtas CTAs per SM
// (8 x 256 threads leave 32 registers per thread, 6 leave 40).  Blocks of at most 65 536 bytes, no dictionary.
template <int kM, int kE, int kTagBits, int kCtas>
__global__ void __launch_bounds__((kM + kE) * 32, kCtas)
lz4_compress_blocks_gnib(BatchArgs a, uint32_t *tickets, uint16_t *gtab)
{
    constexpr int kR = kM / kE;
    static_assert(kM % kE == 0, "every emitter serves the same number of matchers");
    __shared__ __align__(16) uint32_t nt_s[kM * 4096 * kTagBits / 32];
    __shared__ __align__(16) uint4 q_s[kM * 2 * kSeqBatchEntries];
    __shared__ uint32_t meta_s[kM * 8];
    __shared__ __align__(8) uint64_t bars_s[kM * 4];
    __shared__ EmitState st_s[kM];
    const uint32_t warp = threadIdx.x >> 5, lane = lane_id();
    if (threadIdx.x < (uint32_t)kM * 4u) mbar_init(bars_s + threadIdx.x, 1u);
    __syncthreads();
    if (warp >= (uint32_t)kM) {
        const uint32_t e = warp - kM;
        emit_loop_multi<kR>(a, q_s + e * kR * 2 * kSeqBatchEntries, meta_s + e * kR * 8, bars_s + e * kR * 4,
                            st_s + e * kR, lane);
        return;
    }
    SeqProducer pr{q_s + warp * 2 * kSeqBatchEntries, meta_s + warp * 8, bars_s + warp * 4, 0u, 0u, 0u, 0u};
    const uint32_t tab_off = opaque32((blockIdx.x * kM + warp) * 8192u);
    const uint32_t nt_sa = opaque32(smem_addr(nt_s) + warp * (4096u * kTagBits / 8u));
    for (uint32_t b = next_ticket(tickets); b < a.nblocks; b = next_ticket(tickets)) {
        const uint32_t n = a.in_len[b];
        if (n > 65536u) continue;                                           // the u32 kernel's block
        const uint32_t fl = a.flags ? a.flags[b] : 0u;
        if ((uint64_t)a.out_cap[b] < max_output_size_dev(n)) {              // compress.rs:338-340
            if (lane == 0) { a.out_len[b] = 0; a.status[b] = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL; }
            continue;
        }
        const bool h5 = (fl & LZ4B200_BLOCK_HASH5_ALWAYS) || n >= 65535u;
        pr.block = b; pr.first = 1;
        WordView view(a.in + a.in_off[b]);
        match_block_nib<kTagBits>(view, n, reinterpret_cast<uint8_t *>(gtab), tab_off, nt_sa, (fl & LZ4B200_BLOCK_CONT) != 0, h5, pr, lane);
    }
    pr.block = kExitBlock; pr.first = 0;
    pr.flush(0, lane);
    retire_warp(tickets, gridDim.x * kM);
}

#endif  // LZ4B200_AB_VARIANTS (gnib kernel)

#ifdef LZ4B200_AB_VARIANTS
// Tagged global tables (kTag, see match_block): kM matchers + kE emitters per CTA, 16 KiB of (tag, position) entries per
// matcher in global memory.  Blocks of at most 65 536 bytes.
template <int kM, int kE>
__global__ void __launch_bounds__((kM + kE) * 32, 2048 / ((kM + kE) * 32))
lz4_compress_blocks_gtag(BatchArgs a, uint32_t *tickets, uint32_t *gtab)
{
    constexpr int kR = kM / kE;
    static_assert(kM % kE == 0, "every emitter serves the same number of matchers");
    __shared__ __align__(16) uint4 q_s[kM * 2 * kSeqBatchEntries];
    __shared__ uint32_t meta_s[kM * 8];
    __shared__ __align__(8) uint64_t bars_s[kM * 4];
    __shared__ EmitState st_s[kM];
    const uint32_t warp = threadIdx.x >> 5, lane = lane_id();
    if (threadIdx.x < (uint32_t)kM * 4u) mbar_init(bars_s + threadIdx.x, 1u);
    __syncthreads();
    if (warp >= (uint32_t)kM) {
        const uint32_t e = warp - kM;
        emit_loop_multi<kR>(a, q_s + e * kR * 2 * kSeqBatchEntries, meta_s + e * kR * 8, bars_s + e * kR * 4,
                            st_s + e * kR, lane);
        return;
    }
    SeqProducer pr{q_s + warp * 2 * kSeqBatchEntries, meta_s + warp * 8, bars_s + warp * 4, 0u, 0u, 0u, 0u};
    matcher_loop<uint32_t, true, true>(a, tickets, gtab + ((size_t)blockIdx.x * kM + warp) * 4096, pr, lane);
    retire_warp(tickets, gridDim.x * kM);
}

#endif  // LZ4B200_AB_VARIANTS

// =============================================================================================
// Half-warp matchers (lz4_compress_blocks_gtab16): TWO chains per matcher warp, 16 lanes each.
// The global-table kernel is bound by instruction issue while its tables stay in L2, not by HBM: a sequence costs ~230 matcher instructions whether its batch needed 1 probe
// or 32.  Here the same instruction stream serves two blocks at once: each half of a warp owns a block, a table and a
// tuple ring, every warp-level primitive runs under the half's mask, and the halves stay in step because the compiler
// reconverges them at the end of every loop (a half that found its match waits while the other finishes its extra
// batch).  A batch is 16 probes (P(hit within 16) = 97 % on JSON, parse statistics in DESIGN.md), so the step rule of
// compress.rs:374-378 (32 probes per stride value) takes two batches per stride.
// =============================================================================================
template <int G>
struct LaneGroup {                               // G = 16 or 8 consecutive lanes of a warp
    static constexpr uint32_t kAll = (1u << G) - 1u;
    uint32_t sub, gshift, gmask;
    __device__ __forceinline__ explicit LaneGroup(uint32_t lane)
        : sub(lane & (G - 1u)), gshift(lane & ~uint32_t(G - 1)), gmask(kAll << (lane & ~uint32_t(G - 1))) {}
    __device__ __forceinline__ uint32_t ballot(bool p) const { return (__ballot_sync(gmask, p) >> gshift) & kAll; }
    __device__ __forceinline__ uint32_t shfl(uint32_t v, uint32_t src) const { return __shfl_sync(gmask, v, (int)src, G); }
    __device__ __forceinline__ uint32_t match_any(uint32_t key) const { return (__match_any_sync(gmask, key) >> gshift) & kAll; }
    __device__ __forceinline__ void sync() const { __syncwarp(gmask); }
};

template <int G>
struct SeqProducerG {                            // SeqProducer for a lane group (all state uniform within the group)
    uint4 *q;
    volatile uint32_t *meta;
    uint64_t *bars;
    uint32_t k, qn, block, first;
    LaneGroup<G> g;
    __device__ __forceinline__ void flush(uint32_t last)
    {
        const uint32_t h = k & 1u;
        if (g.sub == 0) {
            meta[h * 4 + 0] = block;
            meta[h * 4 + 1] = qn;
            meta[h * 4 + 2] = first | (last << 1);
            mbar_arrive(bars + h);
        }
        k++; qn = 0; first = 0;
        if (k >= 2) mbar_wait_producer(bars + 2 + (k & 1u), ((k >> 1) - 1u) & 1u);
        g.sync();
    }
    __device__ __forceinline__ void push(uint32_t anchor, uint32_t mpos, uint32_t dist, uint32_t end)
    {
        if (g.sub == 0) q[(k & 1u) * kSeqBatchEntries + qn] = make_uint4(anchor, mpos, dist, end);
        qn++;
        if (qn == kSeqBatchEntries) flush(0);
    }
    __device__ __forceinline__ void push_final(uint32_t anchor, uint32_t n)
    {
        if (g.sub == 0) q[(k & 1u) * kSeqBatchEntries + qn] = make_uint4(anchor, 0u, 0u, n);
        qn++;
        flush(1);
    }
};

// The search half of compress_internal (compress.rs:318-489) for one block on 16 lanes; u16 table in global memory.
// Same scheme as match_block_view (speculative pre-batch candidates, shuffles / match.any for in-batch slot collisions,
// commit of the executed probes), 16 probes per batch, 16 bytes per extension round.
template <int kG>
__device__ __forceinline__ void match_block_half(const uint8_t *__restrict__ src, uint32_t n, uint16_t *tab, bool cont, bool h5,
                                                 SeqProducerG<kG> &pr, const LaneGroup<kG> &g)
{
    constexpr uint32_t G = kG, kInvalid = 0xffffu, kAll = LaneGroup<kG>::kAll;
    const uint32_t sub = g.sub, lt_mask = (1u << sub) - 1u;
    if (n < 13) {                                               // compress.rs:343-346
        pr.push_final(0, n);
        return;
    }
    const WordView view(src);
    {
        const uint32_t f = cont ? 0xffffffffu : 0u;
        uint4 *t128 = reinterpret_cast<uint4 *>(tab);
#pragma unroll 4
        for (uint32_t i = sub; i < 512u; i += G) tab_fill16<true>(t128 + i, f);
        g.sync();
    }
    const uint32_t last_probe = n - 12, lim = n - 6;
    uint32_t anchor = 0, cur = 0;
    bool ri = false;                                            // T[H(cur-2)] = cur-2 still owed (compress.rs:460-461)
    if (!cont) {                                                // compress.rs:353-359
        uint32_t lo, hi; view.ro5(0, lo, hi);
        const uint32_t s = h5 ? slot_h5(lo, hi) : slot_h4(lo);
        if (sub == 0) tab_put<true>(tab, s, 0u);
        cur = 1;
        g.sync();
    }
    for (;;) {                                                  // one sequence per iteration
        uint32_t base = cur, nbatch = 0, cand, mpos;
        for (;;) {                                              // probe batches: compress.rs:373-439
            const uint32_t stride = nbatch / (32u / G) + 1u;     // 32 probes per step value = 32/G batches
            const uint32_t p = base + sub * stride;
            const bool term = p > last_probe, live = !term;
            uint32_t v4, hi;
            view.ro5(live ? p : 0u, v4, hi);
            if (ri) {
                uint32_t lo2, hi2; view.ro5(cur - 2u, lo2, hi2);
                const uint32_t s2 = h5 ? slot_h5(lo2, hi2) : slot_h4(lo2);
                if (sub == 0) tab_put<true>(tab, s2, cur - 2u);
                g.sync();
                ri = false;
            }
            uint32_t key = h5 ? slot_h5(v4, hi) : slot_h4(v4);
            uint32_t cnd = kInvalid;
            if (live) cnd = tab_get<true>(tab, key); else key = 0x10000u | sub;
            bool chk = live && cnd != kInvalid && p - cnd <= 65535u;
            bool hit = chk & (view.ro4(chk ? cnd : 0u) == v4);
            uint32_t hits = g.ballot(hit);
            const uint32_t terms = (base + (G - 1u) * stride > last_probe) ? g.ballot(term) : 0u;
            const uint32_t w0 = hits ? (uint32_t)__ffs(hits) - 1u : G;
            uint32_t same = 1u << sub;                          // lanes of this batch on my slot (incl. me)
            bool exact = w0 == 0u;
            if (w0 >= 1u && w0 <= 3u) {
                const uint32_t k0 = g.shfl(key, 0), k1 = g.shfl(key, 1), k2 = g.shfl(key, 2);
                const bool clash = (sub >= 1u && key == k0) || (sub >= 2u && key == k1) || (sub >= 3u && key == k2);
                exact = g.ballot(clash && sub <= w0) == 0u;
            }
            if (!exact) {
                same = g.match_any(key);
                const uint32_t prior = same & lt_mask;
                const uint32_t le0 = w0 >= G - 1u ? kAll : ((2u << w0) - 1u);
                if (g.ballot(prior != 0u) & le0) {
                    if (prior) {
                        cnd = base + (31u - __clz(prior)) * stride;          // forwarded in-batch write
                        chk = p - cnd <= 65535u;                             // lanes with a prior are never term lanes
                        hit = chk & (view.ro4(chk ? cnd : 0u) == v4);
                    }
                    hits = g.ballot(hit);
                }
            }
            const uint32_t win = hits ? (uint32_t)__ffs(hits) - 1u : G;
            const uint32_t tfirst = terms ? (uint32_t)__ffs(terms) - 1u : G;
            if (tfirst < win) {                                 // compress.rs:381-384: the rest is literals
                pr.push_final(anchor, n);
                return;
            }
            // commit the table writes of probes 0..win (last writer per slot wins)
            const uint32_t upto = win < G ? win : G - 1u;
            const uint32_t mine = same & ((2u << upto) - 1u);
            if (sub <= upto && (31u - __clz(mine)) == sub) tab_put<true>(tab, key, p);
            g.sync();
            if (win < G) {
                mpos = base + win * stride;
                cand = g.shfl(cnd, win);
                break;
            }
            base += G * stride;
            nbatch++;
        }
        const uint32_t dist = mpos - cand;
        // ---- extension (compress.rs:156-216, :272-287): forward in 4-byte words per lane (4 G bytes per round: a group of 8
        // lanes covers 32 bytes, what the 32-lane matcher covers with bytes), backward in bytes; the first forward round and
        // the backward round share one memory round trip
        const uint32_t room = min(cand, mpos - anchor);
        const bool inb = sub < room;
        uint8_t b1 = 0, b2 = 1;
        if (room) { b1 = view.byte(mpos - (inb ? 1u + sub : 0u)); b2 = view.byte(cand - (inb ? 1u + sub : 0u)); }
        uint32_t end = mpos + 4u;
        bool lim_stop;
        for (;;) {
            const uint32_t pos = end + 4u * sub;
            const bool full = pos + 4u <= lim;                  // this lane's word lies before n - END_OFFSET
            const uint32_t x = view.ro4(full ? pos : 0u) ^ view.ro4(full ? pos - dist : 0u);
            const uint32_t nm = full ? (x ? (uint32_t)(__ffs(x) - 1) >> 3 : 4u) : 0u;
            const uint32_t bad = g.ballot(nm < 4u);
            if (bad) {
                const uint32_t fl = (uint32_t)__ffs(bad) - 1u;
                end += 4u * fl + g.shfl(nm, fl);
                lim_stop = g.shfl(full ? 0u : 1u, fl) != 0u;    // stopped by the limit, not by a differing byte
                break;
            }
            end += 4u * G;
        }
        uint32_t kb = 0;
        if (room) {
            const uint32_t bad = ~g.ballot(inb && b1 == b2) & kAll;
            kb = bad ? (uint32_t)__ffs(bad) - 1u : G;
        }
        if (lim_stop && end < lim) {                            // a word that crossed n - 6: at most 3 more bytes
            const uint32_t q = end + sub;
            const bool ok = sub < 4u && q < lim && view.byte(q < lim ? q : end) == view.byte((q < lim ? q : end) - dist);
            end += (uint32_t)__ffs(~g.ballot(ok) & kAll) - 1u;
        }
        if (kb) {
            mpos -= kb; cand -= kb;
            while (kb == G) {                                   // more than G bytes backwards: rare
                const uint32_t room2 = min(cand, mpos - anchor);
                const bool inb2 = sub < room2;
                const uint8_t c1 = view.byte(mpos - (inb2 ? 1u + sub : 0u)), c2 = view.byte(cand - (inb2 ? 1u + sub : 0u));
                const uint32_t bad = ~g.ballot(inb2 && c1 == c2) & kAll;
                kb = bad ? (uint32_t)__ffs(bad) - 1u : G;
                mpos -= kb; cand -= kb;
            }
        }
        pr.push(anchor, mpos, dist, end);
        anchor = cur = end;
        ri = true;
    }
}

// kM matcher warps (32/G chains each) + kE emitter warps per CTA; 8 KiB u16 table per chain in global memory.
template <int G, int kM, int kE>
__global__ void __launch_bounds__((kM + kE) * 32, 2048 / ((kM + kE) * 32))
lz4_compress_blocks_gtabg(BatchArgs a, uint32_t *tickets, uint16_t *gtab)
{
    constexpr int kC = (32 / G) * kM, kR = kC / kE;            // chains per CTA, rings per emitter
    static_assert(kC % kE == 0, "every emitter serves the same number of chains");
    __shared__ __align__(16) uint4 q_s[kC * 2 * kSeqBatchEntries];
    __shared__ uint32_t meta_s[kC * 8];
    __shared__ __align__(8) uint64_t bars_s[kC * 4];
    __shared__ EmitState st_s[kC];
    const uint32_t warp = threadIdx.x >> 5, lane = lane_id();
    if (threadIdx.x < (uint32_t)kC * 4u) mbar_init(bars_s + threadIdx.x, 1u);
    __syncthreads();
    if (warp >= (uint32_t)kM) {
        const uint32_t e = warp - kM;
        emit_loop_multi<kR>(a, q_s + e * kR * 2 * kSeqBatchEntries, meta_s + e * kR * 8, bars_s + e * kR * 4,
                            st_s + e * kR, lane);
        return;
    }
    const LaneGroup<G> g(lane);
    const uint32_t chain = warp * (32u / G) + lane / G;
    SeqProducerG<G> pr{q_s + chain * 2 * kSeqBatchEntries, meta_s + chain * 8, bars_s + chain * 4, 0u, 0u, 0u, 0u, g};
    uint16_t *tab = gtab + ((size_t)blockIdx.x * kC + chain) * 4096;
    for (;;) {
        uint32_t b = 0;
        if (g.sub == 0) b = atomicAdd(&tickets[0], 1u);
        b = g.shfl(b, 0);
        if (b >= a.nblocks) break;
        const uint32_t n = a.in_len[b];
        if (n > 65536u) continue;                               // blocks above 64 KiB belong to the u32-table kernel
        const uint32_t fl = a.flags ? a.flags[b] : 0u;
        if ((uint64_t)a.out_cap[b] < max_output_size_dev(n)) {              // compress.rs:338-340
            if (g.sub == 0) { a.out_len[b] = 0; a.status[b] = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL; }
            continue;
        }
        const bool h5 = (fl & LZ4B200_BLOCK_HASH5_ALWAYS) || n >= 65535u;
        pr.block = b; pr.first = 1;
        match_block_half<G>(a.in + a.in_off[b], n, tab, (fl & LZ4B200_BLOCK_CONT) != 0, h5, pr, g);
    }
    pr.block = kExitBlock; pr.first = 0;
    pr.flush(0);
    if (g.sub == 0) {
        __threadfence();
        if (atomicAdd(&tickets[1], 1u) == gridDim.x * kC - 1u) {
            tickets[0] = 0;
            tickets[1] = 0;
            __threadfence();
        }
    }
}

#ifdef LZ4B200_AB_VARIANTS   // measured and rejected (DESIGN.md §6): A/B build only
// ---------------------------------------------------------------------------------------------
// Lane-group matcher with shared-memory tags (lz4_compress_blocks_gtagg): match_block_half's G-lane batches (32/G
// chains per instruction stream: the cheapest instructions per sequence of all the matchers) + match_block_nib's tag
// filter and first-2 verification (no speculative table / candidate traffic, which is what made 16 384 lane-group chains
// thrash the L2).  Tags are 2 bits (1 KiB per chain) so that 112 chains per SM fit.  A batch covers probes
// gi .. gi+G-1 of the current 32-probe step group and never crosses it.  Model: tests/test_warp_emulation.py::warp_encode_nib(G=..).
// ---------------------------------------------------------------------------------------------
template <int kG, int kTagBits>
__device__ __forceinline__ void match_block_group_tag(const uint8_t *__restrict__ src, uint32_t n, uint8_t *gtab, uint32_t tab_off,
                                                      uint32_t nt_sa, bool cont, bool h5, SeqProducerG<kG> &pr, const LaneGroup<kG> &g)
{
    constexpr uint32_t G = kG, kInvalid = 0xffffu, kAll = LaneGroup<kG>::kAll;
    const uint32_t sub = g.sub, lt_mask = (1u << sub) - 1u;
    if (n < 13) {                                               // compress.rs:343-346
        pr.push_final(0, n);
        return;
    }
    const WordView view(src);
    {
        const uint32_t f = cont ? 0xffffffffu : 0u;
        uint4 *t128 = reinterpret_cast<uint4 *>(gtab + tab_off);
#pragma unroll 4
        for (uint32_t i = sub; i < 512u; i += G)
            asm volatile("st.global.cg.v4.u32 [%0], {%1, %1, %1, %1};" ::"l"(t128 + i), "r"(f) : "memory");
        uint32_t lo0, hi0; view.ro5(0, lo0, hi0);               // an empty slot is a candidate at position 0: its tag
        const uint32_t t = tag_fill_word<kTagBits>(tagof<kTagBits>(lo0));
#pragma unroll
        for (uint32_t i = sub; i < 4096u * kTagBits / 8u / 16u; i += G)
            asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(nt_sa + i * 16u), "r"(t) : "memory");
        g.sync();
    }
    const uint32_t last_probe = n - 12, lim = n - 6;
    uint32_t anchor = 0, cur = 0;
    bool ri = false;                                            // T[H(cur-2)] = cur-2 still owed (compress.rs:460-461)
    if (!cont) {                                                // compress.rs:353-359
        uint32_t lo, hi; view.ro5(0, lo, hi);
        const uint32_t s = h5 ? slot_h5(lo, hi) : slot_h4(lo);
        if (sub == 0) { gpos_put(gtab, tab_off, s, 0u); tag_put<kTagBits>(nt_sa, s, tagof<kTagBits>(lo)); }
        cur = 1;
        g.sync();
    }
    for (;;) {                                                  // one sequence per iteration
        uint32_t gbase = cur, stride = 1, gi = 0, cand, mpos;
        for (;;) {                                              // probe batches: compress.rs:373-439
            const uint32_t width = min(G, 32u - gi);
            const uint32_t base = gbase + gi * stride;
            const uint32_t p = base + sub * stride;
            const bool act = sub < width;
            const bool term = act && p > last_probe, live = act && !term;
            uint32_t v4, hi;
            view.ro5(live ? p : 0u, v4, hi);
            if (ri) {
                uint32_t lo2, hi2; view.ro5(cur - 2u, lo2, hi2);
                const uint32_t s2 = h5 ? slot_h5(lo2, hi2) : slot_h4(lo2);
                if (sub == 0) { gpos_put(gtab, tab_off, s2, cur - 2u); tag_put<kTagBits>(nt_sa, s2, tagof<kTagBits>(lo2)); }
                g.sync();
                ri = false;
            }
            uint32_t key = h5 ? slot_h5(v4, hi) : slot_h4(v4);
            const uint32_t mytag = tagof<kTagBits>(v4);
            bool tm = false;
            if (live) tm = tag_get<kTagBits>(nt_sa, key) == mytag; else key = 0x10000u | sub;
            uint32_t pend = g.ballot(tm);
            uint32_t cnd = kInvalid, hits = 0;
            bool hit = false;
            while (pend) {                                      // verify the tag-matching probes two at a time, in order
                const uint32_t rest = pend & (pend - 1u), rest2 = rest & (rest - 1u);
                const bool sel = ((pend & ~rest2) >> sub) & 1u;
                if (sel) {
                    cnd = gpos_get(gtab, tab_off, key);
                    const bool chk = cnd != kInvalid && p - cnd <= 65535u;
                    hit = chk && view.ro4(chk ? cnd : 0u) == v4;
                }
                hits = g.ballot(sel && hit);
                if (hits) break;
                pend = rest2;
            }
            const uint32_t terms = (gbase + 31u * stride > last_probe) ? g.ballot(term) : 0u;
            const uint32_t w0 = hits ? (uint32_t)__ffs(hits) - 1u : G;
            const uint32_t upto0 = w0 < width ? w0 : width - 1u;
            uint32_t same = 1u << sub, win = w0;
            bool exact = w0 == 0u;
            if (w0 >= 1u && w0 <= 3u) {
                const uint32_t k0 = g.shfl(key, 0), k1 = g.shfl(key, 1), k2 = g.shfl(key, 2);
                const bool clash = (sub >= 1u && key == k0) || (sub >= 2u && key == k1) || (sub >= 3u && key == k2);
                exact = g.ballot(clash && sub <= w0) == 0u;
            }
            if (!exact) {
                same = g.match_any(key);
                const uint32_t prior = same & lt_mask;
                const uint32_t le0 = (2u << upto0) - 1u;                     // upto0 <= G - 1 <= 15
                if (g.ballot(prior != 0u) & le0) {
                    const uint32_t pl = prior ? 31u - __clz(prior) : sub;    // the forwarded candidate is a probe of this
                    const uint32_t pv = g.shfl(v4, pl);                      // batch: its 4 bytes sit in that lane's register
                    if (prior) { cnd = base + pl * stride; hit = pv == v4; }
                    const uint32_t h2 = g.ballot(hit) & le0;
                    win = h2 ? (uint32_t)__ffs(h2) - 1u : G;
                }
            }
            const bool partial = win == G && w0 < G;            // forwarding took the hit away: probes 0..w0 were executed
            const uint32_t tfirst = terms ? (uint32_t)__ffs(terms) - 1u : G;
            if (!partial && tfirst < win) {                     // compress.rs:381-384: the rest is literals
                pr.push_final(anchor, n);
                return;
            }
            const uint32_t upto = partial ? w0 : (win < G ? win : width - 1u);
            const uint32_t mine = same & ((2u << upto) - 1u);
            if (sub <= upto && (31u - __clz(mine)) == sub) { gpos_put(gtab, tab_off, key, p); tag_put<kTagBits>(nt_sa, key, mytag); }
            g.sync();
            if (win < G) {
                mpos = base + win * stride;
                cand = g.shfl(cnd, win);
                break;
            }
            gi += upto + 1u;
            if (gi == 32u) { gbase += 32u * stride; stride++; gi = 0; }
        }
        const uint32_t dist = mpos - cand;
        // ---- extension: as match_block_half (forward in 4-byte words per lane, backward in bytes)
        const uint32_t room = min(cand, mpos - anchor);
        const bool inb = sub < room;
        uint8_t b1 = 0, b2 = 1;
        if (room) { b1 = view.byte(mpos - (inb ? 1u + sub : 0u)); b2 = view.byte(cand - (inb ? 1u + sub : 0u)); }
        uint32_t end = mpos + 4u;
        bool lim_stop;
        for (;;) {
            const uint32_t pos = end + 4u * sub;
            const bool full = pos + 4u <= lim;                  // this lane's word lies before n - END_OFFSET
            const uint32_t x = view.ro4(full ? pos : 0u) ^ view.ro4(full ? pos - dist : 0u);
            const uint32_t nm = full ? (x ? (uint32_t)(__ffs(x) - 1) >> 3 : 4u) : 0u;
            const uint32_t bad = g.ballot(nm < 4u);
            if (bad) {
                const uint32_t fl = (uint32_t)__ffs(bad) - 1u;
                end += 4u * fl + g.shfl(nm, fl);
                lim_stop = g.shfl(full ? 0u : 1u, fl) != 0u;    // stopped by the limit, not by a differing byte
                break;
            }
            end += 4u * G;
        }
        uint32_t kb = 0;
        if (room) {
            const uint32_t bad = ~g.ballot(inb && b1 == b2) & kAll;
            kb = bad ? (uint32_t)__ffs(bad) - 1u : G;
        }
        if (lim_stop && end < lim) {                            // a word that crossed n - 6: at most 3 more bytes
            const uint32_t q = end + sub;
            const bool ok = sub < 4u && q < lim && view.byte(q < lim ? q : end) == view.byte((q < lim ? q : end) - dist);
            end += (uint32_t)__ffs(~g.ballot(ok) & kAll) - 1u;
        }
        if (kb) {
            mpos -= kb; cand -= kb;
            while (kb == G) {                                   // more than G bytes backwards: rare
                const uint32_t room2 = min(cand, mpos - anchor);
                const bool inb2 = sub < room2;
                const uint8_t c1 = view.byte(mpos - (inb2 ? 1u + sub : 0u)), c2 = view.byte(cand - (inb2 ? 1u + sub : 0u));
                const uint32_t bad = ~g.ballot(inb2 && c1 == c2) & kAll;
                kb = bad ? (uint32_t)__ffs(bad) - 1u : G;
                mpos -= kb; cand -= kb;
            }
        }
        pr.push(anchor, mpos, dist, end);
        anchor = cur = end;
        ri = true;
    }
}

// kM matcher warps (32/G chains each) + kE emitter warps per CTA, kCtas CTAs per SM; per chain an 8 KiB u16 position
// table in global memory and 4096 x kTagBits bits of tags in shared memory.
template <int G, int kM, int kE, int kTagBits, int kCtas>
__global__ void __launch_bounds__((kM + kE) * 32, kCtas)
lz4_compress_blocks_gtagg(BatchArgs a, uint32_t *tickets, uint16_t *gtab)
{
    constexpr int kC = (32 / G) * kM, kR = kC / kE;            // chains per CTA, rings per emitter
    static_assert(kC % kE == 0, "every emitter serves the same number of chains");
    __shared__ __align__(16) uint32_t nt_s[kC * 4096 * kTagBits / 32];
    __shared__ __align__(16) uint4 q_s[kC * 2 * kSeqBatchEntries];
    __shared__ uint32_t meta_s[kC * 8];
    __shared__ __align__(8) uint64_t bars_s[kC * 4];
    __shared__ EmitState st_s[kC];
    const uint32_t warp = threadIdx.x >> 5, lane = lane_id();
    if (threadIdx.x < (uint32_t)kC * 4u) mbar_init(bars_s + threadIdx.x, 1u);
    __syncthreads();
    if (warp >= (uint32_t)kM) {
        const uint32_t e = warp - kM;
        emit_loop_multi<kR>(a, q_s + e * kR * 2 * kSeqBatchEntries, meta_s + e * kR * 8, bars_s + e * kR * 4,
                            st_s + e * kR, lane);
        return;
    }
    const LaneGroup<G> g(lane);
    const uint32_t chain = warp * (32u / G) + lane / G;
    SeqProducerG<G> pr{q_s + chain * 2 * kSeqBatchEntries, meta_s + chain * 8, bars_s + chain * 4, 0u, 0u, 0u, 0u, g};
    const uint32_t tab_off = opaque32((blockIdx.x * kC + chain) * 8192u);
    const uint32_t nt_sa = opaque32(smem_addr(nt_s) + chain * (4096u * kTagBits / 8u));
    for (;;) {
        uint32_t b = 0;
        if (g.sub == 0) b = atomicAdd(&tickets[0], 1u);
        b = g.shfl(b, 0);
        if (b >= a.nblocks) break;
        const uint32_t n = a.in_len[b];
        if (n > 65536u) continue;                               // blocks above 64 KiB belong to the u32-table kernel
        const uint32_t fl = a.flags ? a.flags[b] : 0u;
        if ((uint64_t)a.out_cap[b] < max_output_size_dev(n)) {              // compress.rs:338-340
            if (g.sub == 0) { a.out_len[b] = 0; a.status[b] = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL; }
            continue;
        }
        const bool h5 = (fl & LZ4B200_BLOCK_HASH5_ALWAYS) || n >= 65535u;
        pr.block = b; pr.first = 1;
        match_block_group_tag<G, kTagBits>(a.in + a.in_off[b], n, reinterpret_cast<uint8_t *>(gtab), tab_off, nt_sa,
                                           (fl & LZ4B200_BLOCK_CONT) != 0, h5, pr, g);
    }
    pr.block = kExitBlock; pr.first = 0;
    pr.flush(0);
    if (g.sub == 0) {
        __threadfence();
        if (atomicAdd(&tickets[1], 1u) == gridDim.x * kC - 1u) {
            tickets[0] = 0;
            tickets[1] = 0;
            __threadfence();
        }
    }
}

#endif  // LZ4B200_AB_VARIANTS (gtagg)

template <typename TabT, int kPairs>
constexpr size_t split_smem_bytes() { return (size_t)kPairs * (4096 * sizeof(TabT) + 2 * kSeqBatchEntries * 16 + kRingBytes + 32 + 32); }

}  // namespace lz4b200
