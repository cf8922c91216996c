// lz4b200_enc_linked.cuh — the linked-frame chain encoder (lz4_compress_frames_linked), included by lz4b200_api.cu.
//
// A BlockMode::Linked frame is one serial chain: lz4_flex's FrameEncoder carries one hash table from block to block
// (frame/compress.rs:261-371), so block k's parse starts from the table block k-1's parse left.  Different frames do not
// depend on each other, so a batch of N linked frames is N chains, and the kernel runs one chain per matcher warp:
//   - a matcher takes a frame by ticket (the host orders frames longest first: a launch lasts as long as its longest
//     chain), zeroes its 16 KiB u32 shared-memory table once, and walks the frame's blocks in order, never refilling the
//     table between blocks and repositioning it where fb::chain_next says (:266-271);
//   - each block is parsed by match_block_linked against the window fb::chain_next gives it (ext_dict, prefix, block);
//   - the sequences go to the matcher's emitter warp through the split encoder's tuple ring, and the emitter writes
//     every block to the slot, out_len and status the block encoders fill, so the frame pipeline after the compressor
//     (block info, scan, gather, checksums, content hash, tail) is the one every frame encoder runs.
// Like match_block_dict, the matcher favours plain code over speed: global loads, full match.any per probe batch.
#pragma once
#include "lz4b200_frame_batch.cuh"
#include "lz4b200_frame_chain.cuh"
#include "lz4b200_kernels.cuh"

namespace lz4b200 {

// One block of a linked frame.  Window coordinates: w[0, ext) is the ext_dict, w[ext, wb) the prefix, w[wb, wb + n) the
// block; they lie back to back in the frame's input.  A table entry is a window coordinate + toff (S - E).  Tuples are
// pushed block-local.
//   - a candidate must be within 65 535 bytes and at or after the window's first byte (compress.rs:403-429);
//   - at or after ext (S): an input candidate, extended backwards to w[ext] and forwards to the block's n - 6;
//   - below ext: an ext_dict candidate, extended backwards to w[0] and forwards to w[ext] at most (:156-170, :272-287).
__device__ __forceinline__ void match_block_linked(const uint8_t *__restrict__ w, uint32_t wb, uint32_t n, uint32_t ext,
                                                   uint32_t toff, bool first, uint32_t *tab, SeqProducer &pr,
                                                   uint32_t lane)
{
    const uint32_t lt_mask = (1u << lane) - 1u;
    if (n < 13) {                                               // compress.rs:343-346
        pr.push_final(0, n, lane);
        return;
    }
    const WordView view(w);
    const uint32_t last_probe = wb + n - 12;
    const uint32_t lim = wb + n - 6;
    uint32_t anchor = wb, cur = wb;
    if (first) {                                                // compress.rs:353-359 (wb == 0, toff == 0)
        uint32_t lo, hi; view.ro5(0, lo, hi);
        if (lane == 0) tab[slot_h5(lo, hi)] = toff;
        cur = 1;
        __syncwarp();
    }
    bool ri = false;
    for (;;) {                                                  // one sequence per iteration
        uint32_t base = cur, stride = 1, cw, mpos;
        for (;;) {                                              // probe batches: compress.rs:373-439
            const uint32_t p = base + lane * stride;
            const bool term = p > last_probe;
            uint32_t v4, hi;
            view.ro5(term ? wb : p, v4, hi);
            if (ri) {                                           // compress.rs:460-461
                uint32_t lo2, hi2; view.ro5(cur - 2u, lo2, hi2);
                if (lane == 0) tab[slot_h5(lo2, hi2)] = cur - 2u + toff;
                __syncwarp();
                ri = false;
            }
            uint32_t key = slot_h5(v4, hi);
            uint32_t cnd = 0;                                   // table coordinate of the candidate
            if (!term) cnd = tab[key]; else key = 0x10000u | lane;
            const uint32_t same = __match_any_sync(kFull, key);
            const uint32_t prior = same & lt_mask;
            if (prior) cnd = toff + base + (31u - __clz(prior)) * stride;   // forwarded in-batch write
            const bool chk = !term && cnd >= toff && p + toff - cnd <= 65535u;
            const bool hit = chk && view.ro4(chk ? cnd - toff : wb) == v4;
            const uint32_t hits = __ballot_sync(kFull, hit), terms = __ballot_sync(kFull, term);
            const uint32_t win = hits ? (uint32_t)__ffs(hits) - 1u : 32u;
            const uint32_t tfirst = terms ? (uint32_t)__ffs(terms) - 1u : 32u;
            if (tfirst < win) {                                 // compress.rs:381-384
                // the probes before the end wrote the table (:391-393), and the frame's next block reads what they wrote
                const uint32_t mine = same & ((1u << tfirst) - 1u);
                if (lane < tfirst && (31u - __clz(mine)) == lane) tab[key] = p + toff;
                __syncwarp();
                pr.push_final(anchor - wb, n, lane);
                return;
            }
            const uint32_t upto = win < 32u ? win : 31u;
            const uint32_t le_mask = upto == 31u ? kFull : ((2u << upto) - 1u);
            const uint32_t mine = same & le_mask;
            if (lane <= upto && (31u - __clz(mine)) == lane) tab[key] = p + toff;
            __syncwarp();
            if (win < 32u) {
                mpos = base + win * stride;
                cw = __shfl_sync(kFull, cnd, win) - toff;
                break;
            }
            base += 32u * stride;
            stride++;
        }
        const uint32_t dist = mpos - cw;
        const bool in_dict = cw < ext;
        const uint32_t src_lo = in_dict ? 0u : ext;             // the candidate's source begins here
        const uint32_t src_hi = in_dict ? ext : 0xffffffffu;    // an ext_dict candidate's source ends at S
        for (;;) {                                              // backwards: compress.rs:272-287
            const uint32_t room = min(cw - src_lo, mpos - anchor);
            const bool inb = lane < room;
            const bool ok = inb && view.byte(mpos - (inb ? 1u + lane : 0u)) == view.byte(cw - (inb ? 1u + lane : 0u));
            const uint32_t bad = ~__ballot_sync(kFull, ok);
            const uint32_t kb = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
            mpos -= kb; cw -= kb;
            if (kb < 32u) break;
        }
        uint32_t end = mpos + 4u, cj = cw + 4u;
        for (;;) {                                              // forwards: compress.rs:156-216 (input and source limits)
            const uint32_t q = end + lane, cq = cj + lane;
            const bool in = q < lim && cq < src_hi;
            const bool ok = in && view.byte(in ? q : mpos) == view.byte(in ? cq : cw);
            const uint32_t bad = ~__ballot_sync(kFull, ok);
            const uint32_t k = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
            end += k; cj += k;
            if (k < 32u) break;
        }
        pr.push(anchor - wb, mpos - wb, dist, end - wb, lane);
        anchor = cur = end;
        ri = true;
    }
}

// Shared memory per matcher/emitter pair: the u32 table, the tuple ring, batch headers and mbarriers (as the split
// encoder's, without its input ring).
constexpr size_t kLinkedPairs = 2;
constexpr size_t kLinkedSmemPerPair = 4096 * sizeof(uint32_t) + 2 * kSeqBatchEntries * 16 + 32 + 32;
constexpr size_t linked_smem_bytes() { return kLinkedPairs * kLinkedSmemPerPair; }

// One CTA = kLinkedPairs matcher warps + as many emitter warps.  order[t] is the frame of ticket t; a's block arrays are
// the ones frame_batch_blocks_kernel writes for the plan.
__global__ void __launch_bounds__(kLinkedPairs * 64)
lz4_compress_frames_linked(BatchArgs a, const fb::FramePlan *plan, const uint32_t *order, uint32_t nframes,
                           uint32_t *tickets)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    constexpr uint32_t kPairs = kLinkedPairs;
    const uint32_t warp = threadIdx.x >> 5, lane = lane_id();
    const uint32_t pair = warp < kPairs ? warp : warp - kPairs;
    constexpr size_t kTab = 4096 * sizeof(uint32_t), kQ = 2 * kSeqBatchEntries * 16;
    uint32_t *tab = reinterpret_cast<uint32_t *>(smem_raw) + pair * 4096;
    uint4 *q = reinterpret_cast<uint4 *>(smem_raw + kPairs * kTab) + pair * 2 * kSeqBatchEntries;
    uint32_t *meta = reinterpret_cast<uint32_t *>(smem_raw + kPairs * (kTab + kQ)) + pair * 8;
    uint64_t *bars0 = reinterpret_cast<uint64_t *>(smem_raw + kPairs * (kTab + kQ + 32));
    uint64_t *bars = bars0 + pair * 4;
    if (threadIdx.x < kPairs * 4u) mbar_init(bars0 + threadIdx.x, 1u);
    __syncthreads();
    if (warp >= kPairs) {
        emit_loop(a, q, meta, bars, lane);
        return;
    }
    SeqProducer pr{q, meta, bars, 0u, 0u, 0u, 0u};
    for (uint32_t t = next_ticket(tickets); t < nframes; t = next_ticket(tickets)) {
        const fb::FramePlan &p = plan[order[t]];
        const uint32_t nb = (uint32_t)fb::frame_blocks(p);
        if (nb == 0) continue;
        {                                                       // a frame opens with an empty table (:244-255)
            uint4 *t128 = reinterpret_cast<uint4 *>(tab);
            for (uint32_t i = lane; i < 1024u; i += 32u) t128[i] = make_uint4(0u, 0u, 0u, 0u);
            __syncwarp();
        }
        fb::ChainState cs = fb::chain_start(p.bs);
        const uint8_t *frame_in = a.in + p.in_off;
        for (uint32_t k = 0; k < nb; k++) {
            const uint32_t b = p.first_block + k;
            const uint32_t n = a.in_len[b];
            const fb::ChainBlock cb = fb::chain_next(cs, n);
            if (cb.reposition) {                                // Table::reposition: saturating subtraction
                const uint32_t shift = (uint32_t)cb.shift;
                for (uint32_t i = lane; i < 4096u; i += 32u) tab[i] = tab[i] > shift ? tab[i] - shift : 0u;
                __syncwarp();
            }
            const uint32_t toff = (uint32_t)(cb.stream - cb.ext_len);
            const uint8_t *w = frame_in + (int64_t)toff + cb.to_frame;
            pr.block = b; pr.first = 1;
            match_block_linked(w, cb.ext_len + cb.prefix, n, cb.ext_len, toff, cb.first, tab, pr, lane);
        }
    }
    pr.block = kExitBlock; pr.first = 0;
    pr.flush(0, lane);
    retire_warp(tickets, gridDim.x * kPairs);
}

}  // namespace lz4b200
