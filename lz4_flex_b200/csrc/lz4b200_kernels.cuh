// lz4b200_kernels.cuh — sm_90a device code of the LZ4 block codec.
//
// K2  lz4_decompress_blocks (+ _linked, _conv)  : decompress_internal  (reference src/block/decompress.rs:201-449)
// K1  lz4_compress_blocks (single warp per block; A/B fallback)     : compress_internal (src/block/compress.rs:318-489)
//     The production encoders — matcher/emitter warp pipelines with shared-memory or global-memory tables —
//     live in lz4b200_enc_split.cuh, included at the end of this file.
//
// All kernels are persistent: a fixed grid of warps pulls block indices from a global ticket
// counter.  This is latency-bound byte shuffling — no tensor cores.  See DESIGN.md for the layout,
// the per-kernel roofline and what each phase costs.
#pragma once
// Build-time variant switches (A/B-measured, see DESIGN.md §experiments).
// ENC_SPLIT=1: matcher warp + emitter warp per block (lz4_compress_blocks_split); 0: one warp does both (v1).
#ifndef ENC_SPLIT
#define ENC_SPLIT 1
#endif
#ifndef ENC_PROBE_NOEMIT
#define ENC_PROBE_NOEMIT 0   // timing probe (invalid output): how much of the chain is emission
#endif
#ifndef DEC_DEFER
#define DEC_DEFER 1
#endif
#ifndef DEC_LIT_PRED
#define DEC_LIT_PRED 1   // 1: fast-path literals as two predicated byte steps instead of a loop; 0: the loop (DESIGN.md §6)
#endif
#ifndef DEC_DEFER8
#define DEC_DEFER8 1     // 1: deferred match stores cover 8 byte steps (64 bytes for G=8); 0: 4 steps (DESIGN.md §6)
#endif
#ifndef DEC_PREFETCH
#define DEC_PREFETCH 0   // > 0: K2 prefetches the compressed stream this many bytes ahead of the token cursor into L1 (build-time A/B)
#endif
#ifndef DEC_DEFER2
#define DEC_DEFER2 0     // 1: TWO short matches in flight (the older one is stored when a third arrives); build-time A/B
#endif
#ifndef DEC_VARIANT_A
#define DEC_VARIANT_A 1
#endif
#ifndef DEC_COPY_UNROLL
#define DEC_COPY_UNROLL 1
#endif

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/lz4b200.h"

namespace lz4b200 {

constexpr uint32_t kFull = 0xffffffffu;

// ---------------------------------------------------------------------------------------------
// descriptors (device pointers)
// ---------------------------------------------------------------------------------------------
struct BatchArgs {
    const uint8_t *in;
    const uint64_t *in_off;
    const uint32_t *in_len;
    const uint8_t *flags;          // compress only; may be null
    uint8_t *out;
    const uint64_t *out_off;
    const uint32_t *out_cap;
    uint32_t *out_len;
    int32_t *status;
    uint64_t *err_expected;        // decompress only; may be null
    uint32_t nblocks;
    uint32_t *tickets;             // [0] next block, [1] warps finished (self-resetting)
    const uint8_t *dict;           // external dictionary shared by every block of the batch (may be null)
    uint32_t dict_len;             // <= 65536: callers keep only the last WINDOW_SIZE bytes
    // BlockMode::Linked frames (lz4_decompress_blocks_linked only): block b may reference the output of the blocks
    // [link_first[b], b) of its frame.  Stored (uncompressed) blocks are not decoded; their bytes are history at
    // in + stored_off[k].  done[] is zeroed by the host and set when a block's output is complete.
    const uint32_t *link_first;
    const uint64_t *stored_off;
    const uint32_t *stored_len;
    uint32_t *done;
};

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

// Pulls the next block index for this warp; the last warp to drain the queue re-arms the
// counters so the next launch needs no memset.
__device__ __forceinline__ uint32_t next_ticket(uint32_t *tickets)
{
    uint32_t t = 0;
    if (lane_id() == 0) t = atomicAdd(&tickets[0], 1u);
    return __shfl_sync(kFull, t, 0);
}
__device__ __forceinline__ void retire_warp(uint32_t *tickets, uint32_t total_warps)
{
    if (lane_id() == 0) {
        __threadfence();
        if (atomicAdd(&tickets[1], 1u) == total_warps - 1) {
            tickets[0] = 0;
            tickets[1] = 0;
            __threadfence();
        }
    }
}

// ---------------------------------------------------------------------------------------------
// unaligned little-endian fetches built from aligned 32-bit loads.
// `w` is the block's base pointer rounded down to 4 bytes, `x` = position + misalignment.
// A fetch of k bytes at x touches only words that contain at least one of those k bytes
// (callers guarantee the k bytes are inside the block), so nothing outside the allocation's
// last touched word is ever read.
// ---------------------------------------------------------------------------------------------
struct WordView {
    const uint32_t *w;
    uint32_t mis;
    __device__ __forceinline__ explicit WordView(const uint8_t *p)
        : w(reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(p) & ~uintptr_t(3))),
          mis(static_cast<uint32_t>(reinterpret_cast<uintptr_t>(p) & 3u)) {}
    // 4 bytes at pos; requires pos+4 <= n and at least one more byte (pos+5 <= n) OR alignment luck:
    // callers use it only where pos + 8 <= n.
    __device__ __forceinline__ uint32_t ro4(uint32_t pos) const
    {
        uint32_t x = pos + mis;
        uint32_t a = __ldg(w + (x >> 2)), b = __ldg(w + (x >> 2) + 1);
        return __funnelshift_r(a, b, (x & 3u) * 8u);
    }
    // ro4 in two steps: ro4_issue(ab, pos, on) loads the two words into ab for lanes with `on` (the other lanes issue no
    // load and keep ab) and ro4_join(ab, pos) makes the 4 bytes of them.  The loads are opaque to the compiler, so two
    // issues under complementary predicates stay two instructions with their own registers: a join of one waits for its
    // lanes' data only.
    __device__ __forceinline__ void ro4_issue(uint2 &ab, uint32_t pos, bool on) const
    {
        const uint32_t *q = w + ((pos + mis) >> 2);
        asm volatile("{ .reg .pred p; setp.ne.u32 p, %3, 0; @p ld.global.nc.u32 %0, [%2]; @p ld.global.nc.u32 %1, [%2+4]; }"
                     : "+r"(ab.x), "+r"(ab.y) : "l"(q), "r"((uint32_t)on));
    }
    __device__ __forceinline__ uint32_t ro4_join(uint2 ab, uint32_t pos) const
    {
        return __funnelshift_r(ab.x, ab.y, ((pos + mis) & 3u) * 8u);
    }
    // 4 bytes at pos; requires only pos + 4 <= n (the second word is fetched only when it holds one of the 4 bytes)
    __device__ __forceinline__ uint32_t ro4s(uint32_t pos) const
    {
        uint32_t x = pos + mis;
        uint32_t a = __ldg(w + (x >> 2)), b = (x & 3u) ? __ldg(w + (x >> 2) + 1) : 0u;
        return __funnelshift_r(a, b, (x & 3u) * 8u);
    }
    // low 5 bytes at pos as (lo32, hi8); requires pos + 8 <= n.
    __device__ __forceinline__ void ro5(uint32_t pos, uint32_t &lo, uint32_t &hi) const
    {
        uint32_t x = pos + mis;
        uint32_t a = __ldg(w + (x >> 2)), b = __ldg(w + (x >> 2) + 1);
        uint32_t sh = (x & 3u) * 8u;
        lo = __funnelshift_r(a, b, sh);
        hi = (b >> sh) & 0xffu;
    }
    __device__ __forceinline__ uint8_t byte(uint32_t pos) const { return __ldg(reinterpret_cast<const uint8_t *>(w) + mis + pos); }
    // the matcher announces the start of a probe batch / sequence here (a view that stages data reacts; this one reads global memory directly)
    __device__ __forceinline__ void advance(uint32_t) const {}
};

// =============================================================================================
// K2: decode.  A block is decoded by a GROUP of G lanes (G = 32, 16, 8 or 4; 32/G blocks per warp).
// Every lane of a group walks the token chain redundantly (uniform within the group, broadcast loads)
// and the G lanes share the byte copies.  Narrow groups trade copy width for fewer warp-instructions
// per sequence: the parse is ~60 instructions whatever G is, so 32/G blocks per warp-instruction
// stream divide the issue cost per sequence, which is what bounds this kernel (see DESIGN.md).
// Semantics = the checked path of decompress_internal (decompress.rs:330-444): same bytes, same
// first error, same OutputTooSmall{expected, actual} fields.
// =============================================================================================
__device__ __forceinline__ void prefetch_global_l1(const void *p)
{
    asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
}

struct DecResult {
    uint32_t written;
    int32_t status;
    uint64_t expected;
};

// out[0..len) = out[-dist ..) with LZ77 byte-serial semantics (duplicate(), duplicate_overlapping():
// decompress.rs:11-82; offset 1 = run fill, decompress_safe.rs:311-313).  T is uint8_t for bytes, uint32_t for the
// range decoder's marker entries (lz4b200_frame_range.cuh).
template <int G, typename T>
__device__ __forceinline__ void copy_match(T *dst, uint32_t dist, uint32_t len, uint32_t sub, uint32_t gmask)
{
    const T *from = dst - dist;
    if (dist >= len) {                       // source entirely older than this match
#if DEC_COPY_UNROLL
        uint32_t i = sub;
        for (; i + 3 * G < len; i += 4 * G) {
            T a = from[i], b = from[i + G], c = from[i + 2 * G], d = from[i + 3 * G];
            dst[i] = a; dst[i + G] = b; dst[i + 2 * G] = c; dst[i + 3 * G] = d;
        }
        for (; i < len; i += G) dst[i] = from[i];
#else
        for (uint32_t i = sub; i < len; i += G) dst[i] = from[i];
#endif
    } else if (dist >= (uint32_t)G) {        // each G-byte step only needs earlier steps
        for (uint32_t base = 0; base < len; base += G) {
            uint32_t i = base + sub;
            if (i < len) dst[i] = from[i];
            __syncwarp(gmask);
        }
    } else {                                 // period < G: every byte is a copy of the seed period
        uint32_t r = sub % dist, step = (uint32_t)G % dist;
        for (uint32_t i = sub; i < len; i += G) {
            dst[i] = from[r];
            r += step;
            if (r >= dist) r -= dist;
        }
    }
}

// One sequence with every check, byte loads only.  Used for the last bytes of a stream, for long
// length encodings and for anything that might fail.  Returns 0 = continue, 1 = stream finished OK,
// 2 = error (r.status set).
template <int G>
__device__ __forceinline__ int decode_sequence_checked(const uint8_t *__restrict__ src, uint32_t n, uint8_t *dst,
                                                    uint32_t cap, uint32_t &ip_io, uint32_t &op_io, uint32_t sub,
                                                    uint32_t gmask, DecResult &r, const uint8_t *__restrict__ dict = nullptr,
                                                    uint32_t dlen = 0)
{
    uint32_t ip = ip_io, op = op_io;
    const uint32_t tok = __ldg(src + ip++);
    uint64_t lit = tok >> 4;
    if (lit == 15) {                                           // read_integer_ptr: decompress.rs:126-157
        for (;;) {
            if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return 2; }
            uint32_t b = __ldg(src + ip++);
            lit += b;
            if (b != 255) break;
        }
    }
    if (lit) {
        if (lit > (uint64_t)(n - ip)) { r.status = LZ4B200_DEC_LITERAL_OUT_OF_BOUNDS; return 2; }   // :346
        if (lit > (uint64_t)(cap - op)) {                                                           // :349-354
            r.status = LZ4B200_DEC_OUTPUT_TOO_SMALL; r.expected = (uint64_t)op + lit; return 2;
        }
        for (uint32_t i = sub; i < (uint32_t)lit; i += G) dst[op + i] = __ldg(src + ip + i);
        ip += (uint32_t)lit; op += (uint32_t)lit;
    }
    if (ip >= n) { ip_io = ip; op_io = op; return 1; }         // the stream ends after literals: :366
    if (n - ip < 2) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return 2; }                   // :373
    const uint32_t dist = (uint32_t)__ldg(src + ip) | ((uint32_t)__ldg(src + ip + 1) << 8);
    ip += 2;
    if (dist == 0) { r.status = LZ4B200_DEC_OFFSET_ZERO; return 2; }                               // :161-173
    uint64_t mlen = 4u + (tok & 15u);
    if (mlen == 19) {
        for (;;) {
            if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return 2; }
            uint32_t b = __ldg(src + ip++);
            mlen += b;
            if (b != 255) break;
        }
    }
    if (dist > op + dlen) { r.status = LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS; return 2; }               // :399
    if (mlen > (uint64_t)(cap - op)) {                                                             // :402-406
        r.status = LZ4B200_DEC_OUTPUT_TOO_SMALL; r.expected = (uint64_t)op + mlen; return 2;
    }
    uint32_t m = (uint32_t)mlen;
    if (dist > op) {
        // the match starts in the external dictionary (copy_from_dict, decompress.rs:85-109): its first
        // dist - op bytes are the dictionary's tail; whatever is left continues at the start of the output
        const uint32_t from_dict = min(m, dist - op);
        const uint8_t *d = dict + (dlen + op - dist);
        for (uint32_t i = sub; i < from_dict; i += G) dst[op + i] = __ldg(d + i);
        op += from_dict; m -= from_dict;
    }
    __syncwarp(gmask);                                         // earlier stores of this group -> visible
    if (m) copy_match<G>(dst + op, dist, m, sub, gmask);
    op += m;
    if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return 2; }                       // :439-443
    ip_io = ip; op_io = op;
    return 0;
}

#ifdef LZ4B200_AB_VARIANTS
// Decodes one block with G lanes.  The token chain is walked kSeqBatch sequences ahead; the byte
// copies of those sequences are then issued together: all literal runs and every match whose source
// lies entirely before the batch (the common case: SURVEY.md §7.2, DESIGN.md "K2") are loaded
// back-to-back and stored afterwards, so one L2/HBM round trip serves the whole batch instead of one
// per sequence.  Matches that read bytes produced inside the batch, overlapping matches and long
// matches run afterwards, in stream order.
constexpr int kSeqBatch = 4;

template <int G>
__device__ __forceinline__ DecResult decode_block(const uint8_t *__restrict__ src, uint32_t n, uint8_t *dst,
                                                  uint32_t cap, uint32_t sub, uint32_t gmask,
                                                  const uint8_t *__restrict__ dict, uint32_t dlen)
{
    constexpr int K = kSeqBatch;
    constexpr int LJ = (14 + G - 1) / G;          // byte steps for a literal run of at most 14
    constexpr int MJ = 4;                         // byte steps for a "short" match (<= 4*G bytes)
    DecResult r{0u, LZ4B200_OK, 0ull};
    if (n == 0) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }   // decompress.rs:207-209
    const WordView view(src);
    uint32_t ip = 0, op = 0;

    for (;;) {
        // ---- phase A: walk up to K sequences that need no check beyond what is tested here ------
        uint32_t s_lsrc[K], s_lit[K], s_dst[K], s_dist[K], s_mlen[K];
        const uint32_t batch_op = op;
        int cnt = 0;
#pragma unroll
        for (int k = 0; k < K; k++) {
            s_lit[k] = 0; s_mlen[k] = 0; s_dist[k] = 1; s_dst[k] = op; s_lsrc[k] = ip;
            if (cnt == k && ip + 8 <= n) {
                const uint32_t v0 = view.ro4(ip);              // token + (if no literals) offset + ext byte
                const uint32_t lit = (v0 >> 4) & 15u;
                const uint32_t q = ip + 1 + lit;               // position of the offset
                if (lit != 15 && q + 8 <= n) {
                    uint32_t v1 = v0 >> 8;
                    if (lit) v1 = view.ro4(q);
                    const uint32_t dist = v1 & 0xffffu;
                    uint32_t mlen = 4u + (v0 & 15u), adv = 2;
                    if (mlen == 19) { mlen += (v1 >> 16) & 0xffu; adv = 3; }
                    const uint32_t at = op + lit;              // output position of the match
                    if (mlen != 19 + 255 && lit + mlen <= cap - op && dist != 0 && dist <= at) {
                        s_lsrc[k] = ip + 1; s_lit[k] = lit; s_dst[k] = at; s_dist[k] = dist; s_mlen[k] = mlen;
                        ip = q + adv;                          // < n because q + 8 <= n
                        op = at + mlen;
                        cnt = k + 1;
                    }
                }
            }
        }
        // ---- phase B: loads.  Slots beyond cnt have lit = mlen = 0 and load nothing. -------------
        uint8_t lv[K][LJ], mv[K][MJ];
        bool later[K];
#pragma unroll
        for (int k = 0; k < K; k++) {
#pragma unroll
            for (int j = 0; j < LJ; j++) {
                const uint32_t i = sub + j * G;
                lv[k][j] = 0;
                if (i < s_lit[k]) lv[k][j] = __ldg(src + s_lsrc[k] + i);
            }
        }
        __syncwarp(gmask);                        // stores of the previous batch -> visible to every lane
#pragma unroll
        for (int k = 0; k < K; k++) {
            // independent of this batch: source ends at or before the batch's first output byte
            const bool indep = s_dst[k] - s_dist[k] + s_mlen[k] <= batch_op;
            later[k] = s_mlen[k] != 0 && !(indep && s_mlen[k] <= (uint32_t)(MJ * G));
            const uint8_t *from = dst + s_dst[k] - s_dist[k];
#pragma unroll
            for (int j = 0; j < MJ; j++) {
                const uint32_t i = sub + j * G;
                mv[k][j] = 0;
                if (!later[k] && i < s_mlen[k]) mv[k][j] = from[i];
            }
        }
        // ---- phase C: stores --------------------------------------------------------------------
#pragma unroll
        for (int k = 0; k < K; k++) {
            uint8_t *lto = dst + s_dst[k] - s_lit[k];
#pragma unroll
            for (int j = 0; j < LJ; j++) {
                const uint32_t i = sub + j * G;
                if (i < s_lit[k]) lto[i] = lv[k][j];
            }
            uint8_t *mto = dst + s_dst[k];
#pragma unroll
            for (int j = 0; j < MJ; j++) {
                const uint32_t i = sub + j * G;
                if (!later[k] && i < s_mlen[k]) mto[i] = mv[k][j];
            }
        }
        // ---- phase D: the matches that had to wait, in stream order -----------------------------
        bool any_later = false;
#pragma unroll
        for (int k = 0; k < K; k++) any_later |= later[k];
        if (any_later) {
#pragma unroll
            for (int k = 0; k < K; k++) {
                if (later[k]) {
                    __syncwarp(gmask);
                    copy_match<G>(dst + s_dst[k], s_dist[k], s_mlen[k], sub, gmask);
                }
            }
        }
        if (cnt == K) continue;
        // ---- the sequence that stopped the walk: every check, one at a time ---------------------
        const int c = decode_sequence_checked<G>(src, n, dst, cap, ip, op, sub, gmask, r, dict, dlen);
        if (c == 1) break;
        if (c == 2) return r;
    }
    r.written = op;
    return r;
}

#endif  // LZ4B200_AB_VARIANTS

// Simple walk: one sequence at a time (fast path + checked path).
//
// DEC_DEFER: the stores of a short, non-overlapping match are held back until just before the next
// match is loaded, so the L2/HBM latency of the back-reference read overlaps the next sequence's token
// walk and literal copy instead of stalling the group at the store (the hottest stall in the profile).
template <int G>
__device__ __forceinline__ DecResult decode_block_simple(const uint8_t *__restrict__ src, uint32_t n, uint8_t *dst,
                                                         uint32_t cap, uint32_t sub, uint32_t gmask,
                                                         const uint8_t *__restrict__ dict, uint32_t dlen)
{
    DecResult r{0u, LZ4B200_OK, 0ull};
    if (n == 0) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }   // decompress.rs:207-209
    const WordView view(src);
    uint32_t ip = 0, op = 0;
    // deferral pays for 8-lane groups (8 byte-steps per match with DEC_DEFER8), not for wider ones
    constexpr bool kDefer = DEC_DEFER && G <= 8;
    uint8_t pv0 = 0, pv1 = 0, pv2 = 0, pv3 = 0;                // pending match bytes of this lane
#if DEC_DEFER8
    uint8_t pv4 = 0, pv5 = 0, pv6 = 0, pv7 = 0;
#endif
    uint32_t p_at = 0, p_len = 0;                              // pending match: output position, length (0 = none)
#if DEC_DEFER2
    uint8_t qv0 = 0, qv1 = 0, qv2 = 0, qv3 = 0;                // the OLDER pending match (two in flight)
    uint32_t q_at = 0, q_len = 0;
#define FLUSH_OLDER()                                                          \
    do {                                                                       \
        if (q_len) {                                                           \
            uint8_t *qd = dst + q_at;                                          \
            if (sub < q_len) qd[sub] = qv0;                                    \
            if (sub + G < q_len) qd[sub + G] = qv1;                            \
            if (sub + 2 * G < q_len) qd[sub + 2 * G] = qv2;                    \
            if (sub + 3 * G < q_len) qd[sub + 3 * G] = qv3;                    \
            q_len = 0;                                                         \
        }                                                                      \
    } while (0)
#else
#define FLUSH_OLDER() do { } while (0)
#endif
#if DEC_DEFER8
#define FLUSH_PENDING_HI()                                                     \
            if (sub + 4 * G < p_len) pd[sub + 4 * G] = pv4;                    \
            if (sub + 5 * G < p_len) pd[sub + 5 * G] = pv5;                    \
            if (sub + 6 * G < p_len) pd[sub + 6 * G] = pv6;                    \
            if (sub + 7 * G < p_len) pd[sub + 7 * G] = pv7;
#else
#define FLUSH_PENDING_HI()
#endif
#define FLUSH_PENDING()                                                        \
    do {                                                                       \
        FLUSH_OLDER();                                                         \
        if (kDefer && p_len) {                                                           \
            uint8_t *pd = dst + p_at;                                          \
            if (sub < p_len) pd[sub] = pv0;                                    \
            if (sub + G < p_len) pd[sub + G] = pv1;                            \
            if (sub + 2 * G < p_len) pd[sub + 2 * G] = pv2;                    \
            if (sub + 3 * G < p_len) pd[sub + 3 * G] = pv3;                    \
            FLUSH_PENDING_HI()                                                 \
            p_len = 0;                                                         \
        }                                                                      \
    } while (0)
    for (;;) {
        if (ip + 8 <= n) {
#if DEC_PREFETCH
            // the token walk reads ~5 bytes per sequence: without a prefetch every eighth sequence waits for HBM on its token
            if (sub == 0) prefetch_global_l1(src + min(ip + (uint32_t)DEC_PREFETCH, n - 1u));
#endif
            const uint32_t v0 = view.ro4(ip);                  // token + (if no literals) offset + ext byte
            const uint32_t lit = (v0 >> 4) & 15u;
            const uint32_t q = ip + 1 + lit;                   // position of the offset
            if (lit != 15 && q + 8 <= n) {
                uint32_t v1 = v0 >> 8;
                if (lit) v1 = view.ro4(q);
                const uint32_t dist = v1 & 0xffffu;
                uint32_t mlen = 4u + (v0 & 15u), adv = 2;
                if (mlen == 19) { mlen += (v1 >> 16) & 0xffu; adv = 3; }
                if ((mlen != 19 + 255) && lit + mlen <= cap - op) {
#if DEC_LIT_PRED
                    if (G >= 8) {                              // lit <= 14 here: at most two byte steps, no loop
                        const uint8_t *ls = src + ip + 1;
                        uint8_t *ld = dst + op;
                        uint8_t l0 = 0, l1 = 0;
                        if (sub < lit) l0 = __ldg(ls + sub);
                        if (G < 16 && sub + G < lit) l1 = __ldg(ls + sub + G);
                        if (sub < lit) ld[sub] = l0;
                        if (G < 16 && sub + G < lit) ld[sub + G] = l1;
                        op += lit;
                    } else
#endif
                    if (lit) {
                        for (uint32_t i = sub; i < lit; i += G) dst[op + i] = __ldg(src + ip + 1 + i);
                        op += lit;
                    }
                    if (dist == 0) { r.status = LZ4B200_DEC_OFFSET_ZERO; return r; }
                    if (dist > op) {
                        // the match starts before the output: in the external dictionary (copy_from_dict,
                        // decompress.rs:85-109), or nowhere (decompress.rs:287-289)
                        if (dist > op + dlen) { r.status = LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS; return r; }
                        FLUSH_PENDING();
                        const uint32_t from_dict = min(mlen, dist - op);
                        const uint8_t *d = dict + (dlen + op - dist);
                        for (uint32_t i = sub; i < from_dict; i += G) dst[op + i] = __ldg(d + i);
                        op += from_dict;
                        __syncwarp(gmask);
                        if (mlen > from_dict) copy_match<G>(dst + op, dist, mlen - from_dict, sub, gmask);
                        op += mlen - from_dict;
                        ip = q + adv;
                        continue;
                    }
#if DEC_DEFER2
                    // two in flight: a new short match whose source ends below the oldest unstored byte only retires the
                    // OLDER pending match (its loads were issued two sequences ago); anything else drains both
                    if (kDefer && dist >= mlen && mlen <= 4u * G && p_len &&
                        op - dist + mlen <= (q_len ? q_at : p_at)) {
                        FLUSH_OLDER();
                        qv0 = pv0; qv1 = pv1; qv2 = pv2; qv3 = pv3; q_at = p_at; q_len = p_len; p_len = 0;
                    } else {
                        FLUSH_PENDING();
                    }
#else
                    FLUSH_PENDING();
#endif
                    __syncwarp(gmask);
                    if (kDefer && dist >= mlen && mlen <= (DEC_DEFER8 ? 8u : 4u) * G) {
                        const uint8_t *from = dst + op - dist;
                        if (sub < mlen) pv0 = from[sub];
                        if (sub + G < mlen) pv1 = from[sub + G];
                        if (sub + 2 * G < mlen) pv2 = from[sub + 2 * G];
                        if (sub + 3 * G < mlen) pv3 = from[sub + 3 * G];
#if DEC_DEFER8
                        if (sub + 4 * G < mlen) pv4 = from[sub + 4 * G];
                        if (sub + 5 * G < mlen) pv5 = from[sub + 5 * G];
                        if (sub + 6 * G < mlen) pv6 = from[sub + 6 * G];
                        if (sub + 7 * G < mlen) pv7 = from[sub + 7 * G];
#endif
                        p_at = op; p_len = mlen;
                    } else {
                        copy_match<G>(dst + op, dist, mlen, sub, gmask);
                    }
                    op += mlen;
                    ip = q + adv;                              // < n because q + 8 <= n
                    continue;
                }
            }
        }
        FLUSH_PENDING();
        const int c = decode_sequence_checked<G>(src, n, dst, cap, ip, op, sub, gmask, r, dict, dlen);
        if (c == 1) break;
        if (c == 2) return r;
    }
    FLUSH_PENDING();
#undef FLUSH_PENDING
#undef FLUSH_PENDING_HI
#undef FLUSH_OLDER
    r.written = op;
    return r;
}

// ---------------------------------------------------------------------------------------------
// Linked blocks (frame/decompress.rs:196-222, 277-305).  In BlockMode::Linked a block's matches may reach
// into the earlier output of its frame (the reference keeps a prefix + ext_dict window of >= 64 KiB; offsets are
// 16-bit, so "everything the frame has produced so far" is equivalent).  That makes the blocks of one frame a
// dependency chain: a group decodes its block normally and, the first time an offset reaches before the block,
// waits for the predecessor blocks it needs (tickets are handed out in stream order, so every predecessor is
// already resident and running) and reads their bytes through L2.  Frames are independent of each other.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t wait_block_done(const BatchArgs &a, uint32_t k)
{
    const uint32_t stored = a.stored_len[k];
    if (stored) return stored;
    volatile uint32_t *flag = a.done + k;
    while (*flag == 0u) __nanosleep(200);
    __threadfence();
    return __ldcg(a.out_len + k);
}

template <int G>
__device__ __forceinline__ DecResult decode_block_linked(const BatchArgs &a, uint32_t b, uint32_t sub, uint32_t gmask)
{
    const uint8_t *__restrict__ src = a.in + a.in_off[b];
    const uint32_t n = a.in_len[b], cap = a.out_cap[b], first = a.link_first[b];
    uint8_t *dst = a.out + a.out_off[b];
    DecResult r{0u, LZ4B200_OK, 0ull};
    if (n == 0) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }   // decompress.rs:207-209
    uint32_t ip = 0, op = 0;
    for (;;) {
        const uint32_t tok = __ldg(src + ip++);
        uint64_t lit = tok >> 4;
        if (lit == 15) {                                           // read_integer_ptr: decompress.rs:126-157
            for (;;) {
                if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }
                const uint32_t v = __ldg(src + ip++);
                lit += v;
                if (v != 255) break;
            }
        }
        if (lit) {
            if (lit > (uint64_t)(n - ip)) { r.status = LZ4B200_DEC_LITERAL_OUT_OF_BOUNDS; return r; }
            if (lit > (uint64_t)(cap - op)) {
                r.status = LZ4B200_DEC_OUTPUT_TOO_SMALL; r.expected = (uint64_t)op + lit; return r;
            }
            for (uint32_t i = sub; i < (uint32_t)lit; i += G) dst[op + i] = __ldg(src + ip + i);
            ip += (uint32_t)lit; op += (uint32_t)lit;
        }
        if (ip >= n) break;                                        // the stream ends after literals
        if (n - ip < 2) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }
        const uint32_t dist = (uint32_t)__ldg(src + ip) | ((uint32_t)__ldg(src + ip + 1) << 8);
        ip += 2;
        if (dist == 0) { r.status = LZ4B200_DEC_OFFSET_ZERO; return r; }
        uint64_t mlen = 4u + (tok & 15u);
        if (mlen == 19) {
            for (;;) {
                if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }
                const uint32_t v = __ldg(src + ip++);
                mlen += v;
                if (v != 255) break;
            }
        }
        // locate the match start when it lies before this block: walk back over the frame's earlier blocks
        uint32_t k = b, back = 0, len_k = 0;
        if (dist > op) {
            back = dist - op;
            bool found = false;
            while (k > first) {
                k--;
                len_k = wait_block_done(a, k);
                if (back <= len_k) { found = true; break; }
                back -= len_k;
            }
            if (!found) { r.status = LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS; return r; }   // decompress.rs:287-289 / :399-401
        }
        if (mlen > (uint64_t)(cap - op)) {
            r.status = LZ4B200_DEC_OUTPUT_TOO_SMALL; r.expected = (uint64_t)op + mlen; return r;
        }
        uint32_t m = (uint32_t)mlen;
        while (m && k < b) {                                       // bytes that come from earlier blocks
            const uint8_t *base = a.stored_len[k] ? a.in + a.stored_off[k] : a.out + a.out_off[k];
            const uint32_t c = min(m, back);
            const uint8_t *from = base + (len_k - back);
            for (uint32_t i = sub; i < c; i += G) dst[op + i] = __ldcg(from + i);
            op += c; m -= c;
            k++;
            if (k < b) { len_k = wait_block_done(a, k); back = len_k; }
        }
        __syncwarp(gmask);
        if (m) copy_match<G>(dst + op, dist, m, sub, gmask);
        op += m;
        if (ip >= n) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; return r; }   // may not end on a match
    }
    r.written = op;
    return r;
}

template <int G>
__global__ void __launch_bounds__(4 * 32)
lz4_decompress_blocks_linked(BatchArgs a)
{
    const uint32_t lane = lane_id();
    const uint32_t sub = lane & (G - 1), leader = lane & ~uint32_t(G - 1);
    const uint32_t gmask = G == 32 ? kFull : (((1u << (G & 31)) - 1u) << leader);
    const uint32_t total_groups = gridDim.x * 4 * (32 / G);
    for (;;) {
        uint32_t b = 0;
        if (sub == 0) b = atomicAdd(&a.tickets[0], 1u);
        b = __shfl_sync(gmask, b, leader);
        if (b >= a.nblocks) break;
        if (a.stored_len[b]) continue;                             // stored block: nothing to decode
        DecResult r = decode_block_linked<G>(a, b, sub, gmask);
        __threadfence();                                           // this lane's output bytes -> visible device-wide
        __syncwarp(gmask);
        if (sub == 0) {
            a.out_len[b] = r.status == LZ4B200_OK ? r.written : 0u;
            a.status[b] = r.status;
            if (a.err_expected) a.err_expected[b] = r.expected;
            __threadfence();
            *(volatile uint32_t *)(a.done + b) = 1u;
        }
    }
    if (sub == 0) {
        __threadfence();
        if (atomicAdd(&a.tickets[1], 1u) == total_groups - 1) {
            a.tickets[0] = 0;
            a.tickets[1] = 0;
            __threadfence();
        }
    }
}

// Warps per CTA.  A batch whose warps are all resident at once (<= 32 one-warp CTAs per SM: 16 384 blocks at G=8 are 31.0
// warps per SM on 132 SMs) runs as ONE-warp CTAs: the block scheduler spreads them evenly over the SMs and a finished warp
// frees its slot at once (faster than two or four warps per CTA on JSON and dickens).  Larger batches
// keep DEC_WARPS_PER_CTA warps per CTA (32 CTAs per SM would cap one-warp CTAs at half the warp slots).
#ifndef DEC_WARPS_PER_CTA
#define DEC_WARPS_PER_CTA 4
#endif
constexpr int kDecWarpsPerCta = DEC_WARPS_PER_CTA;

// kDict: the batch has an external dictionary (decompress_into_with_dict); a separate instantiation so that the
// plain kernel's register allocation is untouched (with the dictionary live ptxas spills in the hot loop).
template <int G, int kBatched, bool kDict, int kW = kDecWarpsPerCta>
__global__ void __launch_bounds__(kW * 32)
lz4_decompress_blocks(BatchArgs a)
{
    const uint32_t lane = lane_id();
    const uint32_t sub = lane & (G - 1), leader = lane & ~uint32_t(G - 1);
    const uint32_t gmask = G == 32 ? kFull : (((1u << (G & 31)) - 1u) << leader);
    const uint32_t total_groups = gridDim.x * kW * (32 / G);
    for (;;) {
        uint32_t b = 0;
        if (sub == 0) b = atomicAdd(&a.tickets[0], 1u);
        b = __shfl_sync(gmask, b, leader);
        if (b >= a.nblocks) break;
#ifdef LZ4B200_AB_VARIANTS
        DecResult r = kBatched
            ? decode_block<G>(a.in + a.in_off[b], a.in_len[b], a.out + a.out_off[b], a.out_cap[b], sub, gmask,
                              kDict ? a.dict : nullptr, kDict ? a.dict_len : 0u)
            : decode_block_simple<G>(a.in + a.in_off[b], a.in_len[b], a.out + a.out_off[b], a.out_cap[b], sub, gmask,
                                     kDict ? a.dict : nullptr, kDict ? a.dict_len : 0u);
#else
        static_assert(kBatched == 0, "the batched walk only exists in the A/B build");
        DecResult r = decode_block_simple<G>(a.in + a.in_off[b], a.in_len[b], a.out + a.out_off[b], a.out_cap[b], sub, gmask,
                                             kDict ? a.dict : nullptr, kDict ? a.dict_len : 0u);
#endif
        if (sub == 0) {
            a.out_len[b] = r.status == LZ4B200_OK ? r.written : 0u;
            a.status[b] = r.status;
            if (a.err_expected) a.err_expected[b] = r.expected;
        }
    }
    if (sub == 0) {
        __threadfence();
        if (atomicAdd(&a.tickets[1], 1u) == total_groups - 1) {
            a.tickets[0] = 0;
            a.tickets[1] = 0;
            __threadfence();
        }
    }
}

#ifdef LZ4B200_AB_VARIANTS
// Converged variant of the decoder (A/B: LZ4B200_DEC_CONV=1).  The plain kernel gives each lane group its own
// block loop, so the 32/G groups of a warp drift apart and serialise (21.7 of 32 lanes active per instruction).
// Here the warp runs ONE loop: every iteration each group decodes one sequence of its current block (or fetches a
// new block), and a full-warp vote at the top of the loop is the reconvergence point.  Same per-sequence code,
// same results.
template <int G>
__global__ void __launch_bounds__(kDecWarpsPerCta * 32)
lz4_decompress_blocks_conv(BatchArgs a)
{
    const uint32_t lane = lane_id();
    const uint32_t sub = lane & (G - 1), leader = lane & ~uint32_t(G - 1);
    const uint32_t gmask = G == 32 ? kFull : (((1u << (G & 31)) - 1u) << leader);
    const uint32_t total_groups = gridDim.x * kDecWarpsPerCta * (32 / G);
    const uint8_t *__restrict__ src = nullptr;
    uint8_t *dst = nullptr;
    const uint32_t *vw = nullptr;
    uint32_t vmis = 0, n = 0, cap = 0, ip = 0, op = 0, b = 0;
    bool have = false, dry = false;
    DecResult r{0u, LZ4B200_OK, 0ull};
    uint8_t pv0 = 0, pv1 = 0, pv2 = 0, pv3 = 0;                // pending (deferred) match bytes of this lane
    uint32_t p_at = 0, p_len = 0;
#define CONV_FLUSH()                                                           \
    do {                                                                       \
        if (p_len) {                                                           \
            uint8_t *pd = dst + p_at;                                          \
            if (sub < p_len) pd[sub] = pv0;                                    \
            if (sub + G < p_len) pd[sub + G] = pv1;                            \
            if (sub + 2 * G < p_len) pd[sub + 2 * G] = pv2;                    \
            if (sub + 3 * G < p_len) pd[sub + 3 * G] = pv3;                    \
            p_len = 0;                                                         \
        }                                                                      \
    } while (0)
    for (;;) {
        if (!have && !dry) {
            if (sub == 0) b = atomicAdd(&a.tickets[0], 1u);
            b = __shfl_sync(gmask, b, leader);
            if (b >= a.nblocks) {
                dry = true;
            } else {
                src = a.in + a.in_off[b]; n = a.in_len[b]; dst = a.out + a.out_off[b]; cap = a.out_cap[b];
                vw = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(src) & ~uintptr_t(3));
                vmis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3u);
                ip = 0; op = 0; p_len = 0;
                r.written = 0; r.status = LZ4B200_OK; r.expected = 0;
                have = true;
            }
        }
        if (__all_sync(kFull, dry)) break;                      // the warp's reconvergence point
        if (!have) continue;
        int fin = 0;                                            // 0 = go on, 1 = block finished, 2 = error
        if (n == 0) { r.status = LZ4B200_DEC_EXPECTED_ANOTHER_BYTE; fin = 2; }   // decompress.rs:207-209
        bool fast = false;
        if (!fin && ip + 8 <= n) {
            uint32_t x = ip + vmis;
            const uint32_t v0 = __funnelshift_r(__ldg(vw + (x >> 2)), __ldg(vw + (x >> 2) + 1), (x & 3u) * 8u);
            const uint32_t lit = (v0 >> 4) & 15u;
            const uint32_t q = ip + 1 + lit;
            if (lit != 15 && q + 8 <= n) {
                uint32_t v1 = v0 >> 8;
                if (lit) {
                    x = q + vmis;
                    v1 = __funnelshift_r(__ldg(vw + (x >> 2)), __ldg(vw + (x >> 2) + 1), (x & 3u) * 8u);
                }
                const uint32_t dist = v1 & 0xffffu;
                uint32_t mlen = 4u + (v0 & 15u), adv = 2;
                if (mlen == 19) { mlen += (v1 >> 16) & 0xffu; adv = 3; }
                if ((mlen != 19 + 255) && lit + mlen <= cap - op) {
                    fast = true;
                    if (lit) {
                        for (uint32_t i = sub; i < lit; i += G) dst[op + i] = __ldg(src + ip + 1 + i);
                        op += lit;
                    }
                    if (dist == 0) { r.status = LZ4B200_DEC_OFFSET_ZERO; fin = 2; }
                    else if (dist > op) { r.status = LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS; fin = 2; }
                    else {
                        CONV_FLUSH();
                        __syncwarp(gmask);
                        if (G <= 8 && dist >= mlen && mlen <= 4u * G) {
                            const uint8_t *from = dst + op - dist;
                            if (sub < mlen) pv0 = from[sub];
                            if (sub + G < mlen) pv1 = from[sub + G];
                            if (sub + 2 * G < mlen) pv2 = from[sub + 2 * G];
                            if (sub + 3 * G < mlen) pv3 = from[sub + 3 * G];
                            p_at = op; p_len = mlen;
                        } else {
                            copy_match<G>(dst + op, dist, mlen, sub, gmask);
                        }
                        op += mlen;
                        ip = q + adv;                           // < n because q + 8 <= n
                    }
                }
            }
        }
        if (!fin && !fast) {
            CONV_FLUSH();
            const int c = decode_sequence_checked<G>(src, n, dst, cap, ip, op, sub, gmask, r);
            if (c == 1) { r.written = op; fin = 1; }
            else if (c == 2) fin = 2;
        }
        if (fin) {
            if (sub == 0) {
                a.out_len[b] = r.status == LZ4B200_OK ? r.written : 0u;
                a.status[b] = r.status;
                if (a.err_expected) a.err_expected[b] = r.expected;
            }
            have = false;
        }
    }
#undef CONV_FLUSH
    if (sub == 0) {
        __threadfence();
        if (atomicAdd(&a.tickets[1], 1u) == total_groups - 1) {
            a.tickets[0] = 0;
            a.tickets[1] = 0;
            __threadfence();
        }
    }
}

#endif  // LZ4B200_AB_VARIANTS

// =============================================================================================
// K1: encode one block with one warp — exact emulation of the reference's sequential greedy
// parse.  The next 32 probe positions of the probe loop (compress.rs:373-439) are evaluated by
// the 32 lanes at once; table writes that the sequential loop would have made between two
// probes of the same batch are forwarded with match.any, and only the writes up to the winning
// probe are committed, so the table state after every sequence is identical to the reference's.
// =============================================================================================
template <typename TabT> struct TabTraits;
template <> struct TabTraits<uint16_t> { static constexpr uint32_t kInvalid = 0xffffu; };
template <> struct TabTraits<uint32_t> { static constexpr uint32_t kInvalid = 0xffffffffu; };

__device__ __forceinline__ uint32_t slot_h4(uint32_t v4)                 // hashtable.rs:19-21 then >>4
{
    return (v4 * 2654435761u) >> 20;
}
__device__ __forceinline__ uint32_t slot_h5(uint32_t lo, uint32_t hi8)   // hashtable.rs:27-34 then >>4
{
    // ((v << 24) * 889523592379) >> 52 with v = hi8:lo (40 bits).  Only the top 12 bits of the low
    // 64 product bits are needed: work on the upper 32-bit half.
    const uint32_t p_lo = 0x1BBCDCBBu, p_hi = 0xCFu;          // 889523592379 = 0xCF_1BBCDCBB
    uint32_t a_lo = lo << 24;                                  // (v << 24) low word
    uint32_t a_hi = (lo >> 8) | (hi8 << 24);                   // (v << 24) high word
    uint32_t top = __umulhi(a_lo, p_lo) + a_lo * p_hi + a_hi * p_lo;
    return top >> 20;
}

// length-extension bytes for value v (= len - 15) at dst; returns number of bytes written.
__device__ __forceinline__ uint32_t put_ext(uint8_t *dst, uint32_t v, uint32_t lane)
{
    uint32_t k = v / 255u, rem = v - k * 255u;
    for (uint32_t i = lane; i < k; i += 32) dst[i] = 0xff;
    if (lane == 0) dst[k] = (uint8_t)rem;
    return k + 1;
}

__device__ __forceinline__ uint32_t put_last_literals(uint8_t *dst, const uint8_t *__restrict__ src,
                                                      uint32_t from, uint32_t n, uint32_t lane)
{
    uint32_t len = n - from, o = 1;
    if (lane == 0) dst[0] = (uint8_t)((len < 15 ? len : 15) << 4);
    if (len >= 15) o += put_ext(dst + o, len - 15, lane);
    for (uint32_t i = lane; i < len; i += 32) dst[o + i] = __ldg(src + from + i);
    return o + len;
}

__device__ __forceinline__ void prefetch_l1(const void *p)
{
    asm volatile("prefetch.global.L1 [%0];" ::"l"(p));
}

#ifdef LZ4B200_AB_VARIANTS
// Single-warp encoder (one warp searches and emits); kept selectable (ENC_SPLIT=0) for A/B runs.
template <typename TabT>
__device__ __forceinline__ uint32_t encode_block_v1(const uint8_t *__restrict__ src, uint32_t n, uint8_t *dst,
                                              TabT *tab, bool cont, bool h5)
{
    constexpr uint32_t kInvalid = TabTraits<TabT>::kInvalid;
    const uint32_t lane = lane_id();
    const uint32_t lt_mask = (1u << lane) - 1u;
    uint32_t o = 0;                                             // output cursor
    if (n < 13) return put_last_literals(dst, src, 0, n, lane);  // compress.rs:343-346

    // table: zero for a fresh table (0 is a legal candidate: position 0), "invalid" when the
    // block continues a frame stream (entries of earlier blocks can never match).
    {
        constexpr uint32_t words = 4096 * sizeof(TabT) / 4;
        uint32_t fill = cont ? 0xffffffffu : 0u;
        uint32_t *t32 = reinterpret_cast<uint32_t *>(tab);
        for (uint32_t i = lane; i < words; i += 32) t32[i] = fill;
        __syncwarp();
    }
    const WordView view(src);
    const uint32_t last_probe = n - 12;
    uint32_t anchor = 0, cur = 0;
    if (!cont) {                                                // compress.rs:353-359
        uint32_t lo, hi; view.ro5(0, lo, hi);
        uint32_t s = h5 ? slot_h5(lo, hi) : slot_h4(lo);
        if (lane == 0) tab[s] = 0;
        cur = 1;
        __syncwarp();
    }

    for (;;) {
        // ---- probe batches ----------------------------------------------------------------
        uint32_t base = cur, stride = 1, cand = 0;
        for (;;) {
            uint32_t p = base + lane * stride;
            bool term = p > last_probe;
            uint32_t key = 0x10000u | lane, v4 = 0, cnd = kInvalid;
            if (!term) {
                uint32_t hi; view.ro5(p, v4, hi);
                key = h5 ? slot_h5(v4, hi) : slot_h4(v4);
                cnd = tab[key];
            }
            uint32_t same = __match_any_sync(kFull, key);
            uint32_t prior = same & lt_mask;
            if (prior) cnd = base + (31u - __clz(prior)) * stride;   // forwarded in-batch write
            bool hit = false;
            if (!term && cnd != kInvalid && p - cnd <= 65535u) hit = (view.ro4(cnd) == v4);
            uint32_t hits = __ballot_sync(kFull, hit), terms = __ballot_sync(kFull, term);
            uint32_t win = hits ? (uint32_t)__ffs(hits) - 1u : 32u;
            uint32_t tfirst = terms ? (uint32_t)__ffs(terms) - 1u : 32u;
            if (tfirst < win)                                       // compress.rs:381-384
                return o + put_last_literals(dst + o, src, anchor, n, lane);
            // commit the table writes of probes 0..win (last writer per slot wins)
            uint32_t upto = win < 32 ? win : 31u;
            uint32_t le_mask = upto == 31 ? kFull : ((2u << upto) - 1u);
            uint32_t mine = same & le_mask;
            if (lane <= upto && (31u - __clz(mine)) == lane) tab[key] = (TabT)p;
            __syncwarp();
            if (win < 32) {
                cur = __shfl_sync(kFull, p, win);
                cand = __shfl_sync(kFull, cnd, win);
                break;
            }
            base += 32u * stride;
            stride++;
        }
        const uint32_t dist = cur - cand;

        // ---- extend backwards (compress.rs:272-287) ---------------------------------------
        for (;;) {
            uint32_t room = min(cand, cur - anchor);                // how far both may step back
            bool ok = lane < room && __ldg(src + cur - 1 - lane) == __ldg(src + cand - 1 - lane);
            uint32_t bad = ~__ballot_sync(kFull, ok);
            uint32_t k = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
            cur -= k; cand -= k;
            if (k < 32) break;
        }
        const uint32_t lit = cur - anchor;

        // ---- extend forwards (compress.rs:156-216), limit n - 6 ---------------------------
        cur += 4; cand += 4;
        uint32_t extra = 0;
        {
            const uint32_t lim = n - 6;
            for (;;) {
                uint32_t q = cur + lane;
                bool ok = q < lim && __ldg(src + q) == __ldg(src + cand + lane);
                uint32_t bad = ~__ballot_sync(kFull, ok);
                uint32_t k = bad ? (uint32_t)__ffs(bad) - 1u : 32u;
                extra += k; cur += k; cand += k;
                if (k < 32) break;
            }
        }
        // ---- T[H(cur-2)] = cur-2 (compress.rs:460-461) ------------------------------------
        {
            uint32_t lo, hi; view.ro5(cur - 2, lo, hi);
            uint32_t s = h5 ? slot_h5(lo, hi) : slot_h4(lo);
            if (lane == 0) tab[s] = (TabT)(cur - 2);
            __syncwarp();
        }
#if ENC_PROBE_NOEMIT
        o += 3 + lit + (lit >= 15 ? 1 : 0) + (extra >= 15 ? 1 : 0); anchor = cur; continue;   // timing probe only: no output
#endif
        // ---- emit the sequence (compress.rs:463-486) --------------------------------------
        if (lane == 0) dst[o] = (uint8_t)(((lit < 15 ? lit : 15) << 4) | (extra < 15 ? extra : 15));
        o++;
        if (lit >= 15) o += put_ext(dst + o, lit - 15, lane);
        for (uint32_t i = lane; i < lit; i += 32) dst[o + i] = __ldg(src + anchor + i);
        o += lit;
        if (lane == 0) { dst[o] = (uint8_t)dist; dst[o + 1] = (uint8_t)(dist >> 8); }
        o += 2;
        if (extra >= 15) o += put_ext(dst + o, extra - 15, lane);
        anchor = cur;
    }
}


#endif  // LZ4B200_AB_VARIANTS

__device__ __forceinline__ uint64_t max_output_size_dev(uint32_t n)
{
    return 20ull + ((uint64_t)n * 110ull) / 100ull;
}

#ifdef LZ4B200_AB_VARIANTS
// One CTA = kWarps warps, each with a private 4096-slot table in shared memory.  Blocks of up to
// 65 536 bytes use the TabT=uint16_t instantiation (8 KiB per table), larger ones uint32_t (16 KiB);
// the host launches both over the same ticket space and each instantiation skips the blocks that
// belong to the other.
template <typename TabT, int kWarps>
__global__ void __launch_bounds__(kWarps * 32)
lz4_compress_blocks(BatchArgs a, uint32_t *tickets)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    TabT *tab = reinterpret_cast<TabT *>(smem_raw) + (threadIdx.x >> 5) * 4096;
    const uint32_t total_warps = gridDim.x * kWarps;
    constexpr bool kSmall = sizeof(TabT) == 2;
    for (uint32_t b = next_ticket(tickets); b < a.nblocks; b = next_ticket(tickets)) {
        const uint32_t n = a.in_len[b];
        if ((n <= 65536u) != kSmall) continue;
        const uint32_t fl = a.flags ? a.flags[b] : 0u;
        uint32_t written = 0; int32_t st = LZ4B200_OK;
        if ((uint64_t)a.out_cap[b] < max_output_size_dev(n)) {              // compress.rs:338-340
            st = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
        } else {
            const bool h5 = (fl & LZ4B200_BLOCK_HASH5_ALWAYS) || n >= 65535u;   // compress.rs:559
            written = encode_block_v1<TabT>(a.in + a.in_off[b], n, a.out + a.out_off[b], tab,
                                            (fl & LZ4B200_BLOCK_CONT) != 0, h5);
        }
        if (lane_id() == 0) { a.out_len[b] = written; a.status[b] = st; }
    }
    retire_warp(tickets, total_warps);
}

#endif  // LZ4B200_AB_VARIANTS

}  // namespace lz4b200

#include "lz4b200_enc_split.cuh"
