// lz4b200_solo_kernel.cuh — K1-S: one compress chain per CTA, everything it touches in shared memory.
//
// A batch of a few hundred big blocks (BASELINE config 4: 256 x 4 MiB per GPU) is a few hundred serial chains
// (compress_internal, reference src/block/compress.rs:318-489): there is nothing to run in parallel but the chains
// themselves, so the only lever is the latency of one probe.  Here a chain gets half an SM's shared memory:
//   * its 4096-entry u32 table (16 KiB; hashtable.rs:52-53,121-127),
//   * an 80 KiB ring holding the input window [cursor - 64 KiB, cursor + 12 KiB): every candidate the format allows
//     (MAX_DISTANCE 65 535, block/mod.rs:64) is a shared-memory read, not an L2/HBM round trip,
//   * the ring is filled 2 KiB at a time by TMA bulk copies (cp.async.bulk.shared.global, completion on one mbarrier
//     per ring slot) issued six chunks ahead of the furthest byte the parse has touched.
// The matcher is ONE thread running tc::parse_block_thread (the same sequential parse the K1-T kernel runs per lane)
// over ring views; it hands (anchor, match start, offset, match end) tuples to an emitter warp through the tuple
// queue of lz4b200_enc_split.cuh, and the emitter writes the byte stream with warp-wide scans and coalesced stores
// (emit_batch).  Probe latency: ~100 cycles of LDS + integer work instead of two dependent L2/HBM accesses.
#pragma once
#include "lz4b200_solo_ring.cuh"

namespace lz4b200 {

#ifdef LZ4B200_AB_VARIANTS
// Single-thread producer side of the tuple queue (same protocol as SeqProducer, lz4b200_enc_split.cuh).
struct SoloSink {
    uint4 *q;
    volatile uint32_t *meta;
    uint64_t *bars;            // full[0], full[1], empty[0], empty[1]
    uint32_t k, qn, block, first;
    SoloFeed *feed;

    __device__ __forceinline__ void flush(uint32_t last)
    {
        const uint32_t h = k & 1u;
        meta[h * 4 + 0] = block;
        meta[h * 4 + 1] = qn;
        meta[h * 4 + 2] = first | (last << 1);
        mbar_arrive(bars + h);
        k++; qn = 0; first = 0;
        if (k >= 2) mbar_wait(bars + 2 + (k & 1u), ((k >> 1) - 1u) & 1u);
    }
    __device__ __forceinline__ void sequence(uint32_t anchor, uint32_t mpos, uint32_t dist, uint32_t end)
    {
        q[(k & 1u) * kSeqBatchEntries + qn] = make_uint4(anchor, mpos, dist, end);
        if (++qn == kSeqBatchEntries) flush(0);
        feed->prefetch(end + feed->mis);                   // keep the TMA three chunks ahead of the cursor
    }
    __device__ __forceinline__ void tail(uint32_t anchor, uint32_t n)
    {
        q[(k & 1u) * kSeqBatchEntries + qn] = make_uint4(anchor, 0u, 0u, n);
        qn++;
        flush(1);
    }
};

constexpr size_t kSoloSmemBytes = kSoloRing + 4096 * 4 + 2 * kSeqBatchEntries * 16 + 32 + 4 * 8 + kSoloSlots * 8;

// warp 0, lane 0: matcher; warp 1: emitter.
__global__ void __launch_bounds__(64)
lz4_compress_blocks_solo(BatchArgs a, uint32_t *tickets)
{
    extern __shared__ __align__(128) uint8_t solo_smem[];
    uint8_t *ring = solo_smem;
    uint32_t *tab = reinterpret_cast<uint32_t *>(solo_smem + kSoloRing);
    uint4 *q = reinterpret_cast<uint4 *>(solo_smem + kSoloRing + 16384);
    uint32_t *meta = reinterpret_cast<uint32_t *>(solo_smem + kSoloRing + 16384 + 2 * kSeqBatchEntries * 16);
    uint64_t *bars = reinterpret_cast<uint64_t *>(solo_smem + kSoloRing + 16384 + 2 * kSeqBatchEntries * 16 + 32);
    uint64_t *rbars = bars + 4;
    if (threadIdx.x < 4u + kSoloSlots) mbar_init(bars + threadIdx.x, 1u);
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5, lane = lane_id();
    if (warp == 1u) {
        emit_loop(a, q, meta, bars, lane);
        return;
    }
    if (lane != 0u) return;
    SoloFeed feed;
    feed.ring = ring; feed.bars = rbars; feed.phases = 0ull;
    SoloSink sink{q, meta, bars, 0u, 0u, 0u, 0u, &feed};
    for (;;) {
        const uint32_t b = atomicAdd(&tickets[0], 1u);
        if (b >= a.nblocks) break;
        const uint32_t n = a.in_len[b];
        const uint32_t fl = a.flags ? a.flags[b] : 0u;
        if ((uint64_t)a.out_cap[b] < max_output_size_dev(n)) {              // compress.rs:338-340
            a.out_len[b] = 0; a.status[b] = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
            continue;
        }
        const bool cont = (fl & LZ4B200_BLOCK_CONT) != 0;
        const bool h5 = (fl & LZ4B200_BLOCK_HASH5_ALWAYS) || n >= 65535u;   // compress.rs:559
        {
            const uint32_t f = cont ? 0xffffffffu : 0u;
            uint4 *t128 = reinterpret_cast<uint4 *>(tab);
#pragma unroll 8
            for (uint32_t i = 0; i < 1024u; i++) t128[i] = make_uint4(f, f, f, f);
        }
        feed.begin(a.in + a.in_off[b], n);
        RingStream<true> in;
        RingStream<false> cs;
        in.init(&feed); cs.init(&feed);
        sink.block = b; sink.first = 1;
        tc::parse_block_thread<uint32_t>(in, cs, n, tab, cont, h5, sink);
        feed.drain();
    }
    sink.block = kExitBlock; sink.first = 0;
    sink.flush(0);
    __threadfence();
    if (atomicAdd(&tickets[1], 1u) == gridDim.x - 1u) {
        tickets[0] = 0;
        tickets[1] = 0;
        __threadfence();
    }
}

#endif  // LZ4B200_AB_VARIANTS

// =============================================================================================
// K1-S2: the same idea with the WARP matcher.  The single-thread matcher above pays ~5 cycles per dependent instruction
// with nobody to hide them (hundreds of cycles per probe step); the warp matcher of
// lz4b200_enc_split.cuh evaluates 32 probes per batch and extends 32 bytes per round, so the same dependent latency buys a
// whole sequence.  match_block_view runs unchanged over a view that serves bytes from a shared-memory ring:
//   * 64 KiB ring (power of two: index = x & 0xffff), 32 slots of 2 KiB, filled by TMA bulk copies issued six chunks
//     ahead of the cursor by lane 0; it therefore holds [cursor - ~50 KiB, cursor + 12 KiB);
//   * the ring is a CACHE with an exact validity test (ring_lo <= x < ring_hi): anything outside — candidates further
//     back than the ring reaches, probes of a long stride that run ahead of it, chunks still in flight — is read from
//     global memory like the other kernels do.  Correctness never depends on what the ring holds.
// =============================================================================================
constexpr uint32_t kRing2Chunk = 2048, kRing2Slots = 32, kRing2Bytes = kRing2Chunk * kRing2Slots, kRing2Ahead = 6;

struct WarpRingView {
    const uint32_t *w;         // global fallback: src rounded down to 4 bytes (WordView)
    uint32_t gmis;             // src & 3
    const uint32_t *ring32;    // the ring as words
    uint8_t *ring;
    uint64_t *bars;            // kRing2Slots mbarriers
    const uint8_t *src_al;     // src rounded down to 16 bytes
    uint32_t mis;              // src & 15: ring x space = position + mis
    uint32_t xend, nchunks, issued, waited, phases, lane;
    uint32_t ring_lo, ring_hi; // x range whose bytes are valid in the ring

    __device__ __forceinline__ void begin(const uint8_t *src, uint32_t n, uint32_t lane_)
    {
        w = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(src) & ~uintptr_t(3));
        gmis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3u);
        mis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 15u);
        src_al = src - mis;
        xend = mis + n;
        nchunks = (xend + kRing2Chunk - 1u) / kRing2Chunk;
        issued = waited = 0; ring_lo = ring_hi = 0;
        lane = lane_;
    }
    // The cursor is at block position pos (warp-uniform call): request chunks up to kRing2Ahead past it, and make sure the
    // cursor's chunk and the next one have landed.
    __device__ __forceinline__ void advance(uint32_t pos)
    {
        const uint32_t c = (pos + mis) / kRing2Chunk;
        const uint32_t stop = c + kRing2Ahead + 1u < nchunks ? c + kRing2Ahead + 1u : nchunks;
        if (issued < stop) {
            if (lane == 0) {
                for (uint32_t k = issued; k < stop; k++) {
                    const uint32_t s = k % kRing2Slots, x0 = k * kRing2Chunk;
                    const uint32_t valid = xend - x0 < kRing2Chunk ? xend - x0 : kRing2Chunk;
                    const uint32_t body = valid & ~15u;
                    uint8_t *dst = ring + s * kRing2Chunk;
                    for (uint32_t i = body; i < valid; i++) dst[i] = __ldg(src_al + x0 + i);   // the block's last <16 bytes
                    ring_fill(dst, src_al + x0, body, bars + s);
                }
            }
            issued = stop;
            __syncwarp();
        }
        const uint32_t wc = c + 1u < issued ? c + 1u : issued - 1u;     // issued >= 1 here whenever the block has bytes
        while (waited <= wc && waited < issued) {
            const uint32_t s = waited % kRing2Slots;
            ring_wait(bars + s, (phases >> s) & 1u);
            phases ^= 1u << s;
            waited++;
        }
        ring_lo = issued > kRing2Slots ? (issued - kRing2Slots) * kRing2Chunk : 0u;
        ring_hi = waited * kRing2Chunk;
    }
    __device__ __forceinline__ void drain()                           // every request waited: the slots are reusable
    {
        while (waited < issued) {
            const uint32_t s = waited % kRing2Slots;
            ring_wait(bars + s, (phases >> s) & 1u);
            phases ^= 1u << s;
            waited++;
        }
        __syncwarp();
    }
    __device__ __forceinline__ bool cached(uint32_t x_lo, uint32_t x_hi) const   // bytes [x_lo, x_hi] are in the ring
    {
        return x_lo >= ring_lo && x_hi < ring_hi;
    }
    __device__ __forceinline__ uint32_t ro4(uint32_t pos) const
    {
        const uint32_t x = pos + mis;
        if (cached(x & ~3u, (x & ~3u) + 7u)) {
            const uint32_t a = ring32[(x >> 2) & (kRing2Bytes / 4 - 1u)], b = ring32[((x >> 2) + 1u) & (kRing2Bytes / 4 - 1u)];
            return __funnelshift_r(a, b, (x & 3u) * 8u);
        }
        const uint32_t g = pos + gmis;
        const uint32_t a = __ldg(w + (g >> 2)), b = (g & 3u) ? __ldg(w + (g >> 2) + 1) : 0u;
        return __funnelshift_r(a, b, (g & 3u) * 8u);
    }
    __device__ __forceinline__ void ro5(uint32_t pos, uint32_t &lo, uint32_t &hi) const   // requires pos + 8 <= n
    {
        const uint32_t x = pos + mis;
        uint32_t a, b, sh;
        if (cached(x & ~3u, (x & ~3u) + 7u)) {
            a = ring32[(x >> 2) & (kRing2Bytes / 4 - 1u)]; b = ring32[((x >> 2) + 1u) & (kRing2Bytes / 4 - 1u)];
            sh = (x & 3u) * 8u;
        } else {
            const uint32_t g = pos + gmis;
            a = __ldg(w + (g >> 2)); b = __ldg(w + (g >> 2) + 1);
            sh = (g & 3u) * 8u;
        }
        lo = __funnelshift_r(a, b, sh);
        hi = (b >> sh) & 0xffu;
    }
    __device__ __forceinline__ uint8_t byte(uint32_t pos) const
    {
        const uint32_t x = pos + mis;
        if (cached(x, x)) return ring[x & (kRing2Bytes - 1u)];
        return __ldg(reinterpret_cast<const uint8_t *>(w) + gmis + pos);
    }
};

constexpr size_t kSolo2SmemBytes = kRing2Bytes + 4096 * 4 + 2 * kSeqBatchEntries * 16 + 32 + 4 * 8 + kRing2Slots * 8;

// warp 0: matcher (32 lanes); warp 1: emitter.  u32 table (any block size up to 8 MiB).
__global__ void __launch_bounds__(64)
lz4_compress_blocks_solo2(BatchArgs a, uint32_t *tickets)
{
    extern __shared__ __align__(128) uint8_t solo_smem[];
    uint8_t *ring = solo_smem;
    uint32_t *tab = reinterpret_cast<uint32_t *>(solo_smem + kRing2Bytes);
    uint4 *q = reinterpret_cast<uint4 *>(solo_smem + kRing2Bytes + 16384);
    uint32_t *meta = reinterpret_cast<uint32_t *>(solo_smem + kRing2Bytes + 16384 + 2 * kSeqBatchEntries * 16);
    uint64_t *bars = reinterpret_cast<uint64_t *>(solo_smem + kRing2Bytes + 16384 + 2 * kSeqBatchEntries * 16 + 32);
    uint64_t *rbars = bars + 4;
    if (threadIdx.x < 4u + kRing2Slots) mbar_init(bars + threadIdx.x, 1u);
    __syncthreads();
    const uint32_t warp = threadIdx.x >> 5, lane = lane_id();
    if (warp == 1u) {
        emit_loop(a, q, meta, bars, lane);
        return;
    }
    WarpRingView view;
    view.ring = ring; view.ring32 = reinterpret_cast<const uint32_t *>(ring); view.bars = rbars; view.phases = 0u;
    SeqProducer pr{q, meta, bars, 0u, 0u, 0u, 0u};
    for (uint32_t b = next_ticket(tickets); b < a.nblocks; b = next_ticket(tickets)) {
        const uint32_t n = a.in_len[b];
        const uint32_t fl = a.flags ? a.flags[b] : 0u;
        if ((uint64_t)a.out_cap[b] < max_output_size_dev(n)) {              // compress.rs:338-340
            if (lane == 0) { a.out_len[b] = 0; a.status[b] = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL; }
            continue;
        }
        const bool h5 = (fl & LZ4B200_BLOCK_HASH5_ALWAYS) || n >= 65535u;   // compress.rs:559
        pr.block = b; pr.first = 1;
        view.begin(a.in + a.in_off[b], n, lane);
        match_block_view<uint32_t, false, false>(view, n, tab, nullptr, (fl & LZ4B200_BLOCK_CONT) != 0, h5, pr, lane);
        view.drain();
    }
    pr.block = kExitBlock; pr.first = 0;
    pr.flush(0, lane);
    retire_warp(tickets, gridDim.x);
}

}  // namespace lz4b200
