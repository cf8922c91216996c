// lz4b200_api.cu — host runtime and C ABI (include/lz4b200.h) of the H100 (sm_90a) LZ4 block codec.
//
// Everything here is product code: contexts, launch plumbing, host<->device staging and the
// frame container (header / BlockInfo / checksums), which is host-side bookkeeping around the
// two block kernels.  There is no CPU codec in this library: without a CUDA device every entry
// point that has work to do fails with LZ4B200_CUDA_ERROR.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "lz4b200_kernels.cuh"
#include "lz4b200_solo_kernel.cuh"
#ifdef LZ4B200_AB_VARIANTS
// A/B build (lz4_flex_b200/liblz4b200_ab.so, -DLZ4B200_AB_VARIANTS): the kernels that lost their measurements stay
// compilable and testable there (tests/test_gpu_kernel_variants.py) but are not part of the product library.
#include "lz4b200_thread_kernels.cuh"
#endif

using namespace lz4b200;

// ---------------------------------------------------------------------------------------------
// small device helpers used by the frame path
// ---------------------------------------------------------------------------------------------
namespace lz4b200 {

// Exclusive scan of sizes[0..n) into offs[0..n], offs[n] = total.  One CTA; n is a block count
// (<= a few 100k), so a single-CTA chunked scan is far below launch noise.
__global__ void __launch_bounds__(1024) scan_sizes_kernel(const uint32_t *sizes, uint64_t *offs, uint32_t n)
{
    __shared__ uint64_t warp_sums[32];
    __shared__ uint64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < n; base += 1024) {
        uint32_t i = base + threadIdx.x;
        uint64_t v = i < n ? sizes[i] : 0, x = v;
        for (int d = 1; d < 32; d <<= 1) {
            uint64_t y = __shfl_up_sync(kFull, x, d);
            if ((threadIdx.x & 31) >= d) x += y;
        }
        if ((threadIdx.x & 31) == 31) warp_sums[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint64_t w = warp_sums[threadIdx.x], s = w;
            for (int d = 1; d < 32; d <<= 1) {
                uint64_t y = __shfl_up_sync(kFull, s, d);
                if (threadIdx.x >= d) s += y;
            }
            warp_sums[threadIdx.x] = s - w;
        }
        __syncthreads();
        uint64_t excl = carry + warp_sums[threadIdx.x >> 5] + x - v;
        if (i < n) offs[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) offs[n] = carry;
}

// Generic gather: segment b copies len[b] bytes from src_base[sel] + src_off[b] to dst + dst_off[b],
// optionally preceded by a 4-byte little-endian word (the frame BlockInfo).  One CTA per segment
// slice; byte-granular head/tail, 16-byte body when co-aligned.
struct GatherArgs {
    const uint8_t *src_a;          // segment source when pick[b] == 0
    const uint8_t *src_b;          // segment source when pick[b] != 0
    const uint64_t *off_a;
    const uint64_t *off_b;
    const uint32_t *len_a;
    const uint32_t *len_b;
    const uint8_t *pick;           // may be null (always a)
    const uint32_t *prefix_word;   // may be null; else written as 4 LE bytes before the payload
    uint8_t *dst;
    const uint64_t *dst_off;
    uint32_t nseg;
    const uint64_t *dst_shift = nullptr;   // optional device scalar added to every destination offset
};

__global__ void __launch_bounds__(256) gather_segments_kernel(GatherArgs g)
{
    for (uint32_t b = blockIdx.x; b < g.nseg; b += gridDim.x) {
        const bool second = g.pick && g.pick[b];
        const uint8_t *s = second ? g.src_b + g.off_b[b] : g.src_a + g.off_a[b];
        const uint32_t len = second ? g.len_b[b] : g.len_a[b];
        uint8_t *d = g.dst + g.dst_off[b] + (g.dst_shift ? *g.dst_shift : 0ull);
        if (g.prefix_word) {
            if (threadIdx.x < 4) d[threadIdx.x] = (uint8_t)(g.prefix_word[b] >> (8 * threadIdx.x));
            d += 4;
        }
        const uint32_t dm = (uint32_t)(reinterpret_cast<uintptr_t>(d) & 15u);
        const uint32_t sm = (uint32_t)(reinterpret_cast<uintptr_t>(s) & 15u);
        if (dm == sm && len >= 64) {
            uint32_t head = (16u - dm) & 15u;
            if (threadIdx.x < head) d[threadIdx.x] = s[threadIdx.x];
            uint32_t body = (len - head) >> 4;
            const uint4 *s4 = reinterpret_cast<const uint4 *>(s + head);
            uint4 *d4 = reinterpret_cast<uint4 *>(d + head);
            for (uint32_t i = threadIdx.x; i < body; i += blockDim.x) d4[i] = s4[i];
            uint32_t done = head + (body << 4);
            if (done + threadIdx.x < len) d[done + threadIdx.x] = s[done + threadIdx.x];
        } else {
            for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) d[i] = s[i];
        }
    }
}

// Frame encoder bookkeeping for a block range: per block, decide compressed-vs-stored
// (frame/compress.rs:301-306) and produce BlockInfo word + segment size.
__global__ void frame_block_info_kernel(const uint32_t *comp_len, const uint32_t *raw_len, uint32_t n,
                                        uint32_t *info_word, uint8_t *pick_raw, uint32_t *seg_size,
                                        uint32_t *payload_len)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t c = comp_len[i], r = raw_len[i];
    bool stored = !(c < r);
    info_word[i] = stored ? (r | 0x80000000u) : c;
    pick_raw[i] = stored ? 1 : 0;
    payload_len[i] = stored ? r : c;
    seg_size[i] = 4u + (stored ? r : c);
}

// Descriptor generator for a run of equal-sized blocks cut from one contiguous buffer.
__global__ void make_uniform_desc_kernel(uint64_t total_len, uint32_t block, uint64_t out_stride,
                                         uint64_t first_block, uint64_t fresh_period, uint32_t n,
                                         uint64_t *in_off, uint32_t *in_len, uint64_t *out_off,
                                         uint32_t *out_cap, uint8_t *flags)
{
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t o = (uint64_t)i * block;
    uint64_t rem = total_len - o;
    in_off[i] = o;
    in_len[i] = (uint32_t)(rem < block ? rem : block);
    out_off[i] = (uint64_t)i * out_stride;
    out_cap[i] = (uint32_t)out_stride;
    if (flags) {
        uint64_t k = first_block + i;
        bool fresh = (k % fresh_period) == 0;
        flags[i] = (uint8_t)(LZ4B200_BLOCK_HASH5_ALWAYS | (fresh ? 0u : LZ4B200_BLOCK_CONT));
    }
}

}  // namespace lz4b200

// ---------------------------------------------------------------------------------------------
// XXH32 (host) — header checksum byte, block and content checksums
// ---------------------------------------------------------------------------------------------
namespace {

inline uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline void wr32(uint8_t *p, uint32_t v) { memcpy(p, &v, 4); }
inline uint32_t rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

constexpr uint32_t kP1 = 2654435761u, kP2 = 2246822519u, kP3 = 3266489917u, kP4 = 668265263u, kP5 = 374761393u;

struct Xxh32 {
    uint32_t acc[4];
    uint8_t buf[16];
    uint32_t fill = 0;
    uint64_t total = 0;
    uint32_t seed;
    explicit Xxh32(uint32_t s = 0) : seed(s)
    {
        acc[0] = s + kP1 + kP2; acc[1] = s + kP2; acc[2] = s; acc[3] = s - kP1;
    }
    static uint32_t round(uint32_t a, uint32_t v) { return rotl(a + v * kP2, 13) * kP1; }
    void stripe(const uint8_t *p)
    {
        for (int i = 0; i < 4; i++) acc[i] = round(acc[i], rd32(p + 4 * i));
    }
    void update(const uint8_t *p, size_t n)
    {
        total += n;
        if (fill) {
            size_t take = std::min<size_t>(16 - fill, n);
            memcpy(buf + fill, p, take); fill += (uint32_t)take; p += take; n -= take;
            if (fill < 16) return;
            stripe(buf); fill = 0;
        }
        for (; n >= 16; p += 16, n -= 16) stripe(p);
        if (n) { memcpy(buf, p, n); fill = (uint32_t)n; }
    }
    uint32_t digest() const
    {
        uint32_t h = total >= 16 ? rotl(acc[0], 1) + rotl(acc[1], 7) + rotl(acc[2], 12) + rotl(acc[3], 18)
                                 : seed + kP5;
        h += (uint32_t)total;
        const uint8_t *p = buf, *e = buf + fill;
        for (; p + 4 <= e; p += 4) h = rotl(h + rd32(p) * kP3, 17) * kP4;
        for (; p < e; p++) h = rotl(h + (*p) * kP5, 11) * kP1;
        h ^= h >> 15; h *= kP2; h ^= h >> 13; h *= kP3; h ^= h >> 16;
        return h;
    }
};

size_t block_size_bytes(int id)
{
    switch (id) {
    case 4: return 64u << 10;
    case 5: return 256u << 10;
    case 6: return 1u << 20;
    case 7: return 4u << 20;
    case 8: return 8u << 20;
    default: return 0;
    }
}

// BlockSize::from_buf_length — frame/header.rs:57-67
int auto_block_size_id(size_t first_write_len)
{
    if (first_write_len > (256u << 10)) return 7;
    if (first_write_len > (64u << 10)) return 5;
    return 4;
}

// Number of consecutive full blocks that share one table epoch before FrameEncoder repositions
// its table (frame/compress.rs:266-271): block k is FRESH iff k % period == 0.
uint64_t fresh_period(size_t bs)
{
    // reposition fires at the first block whose starting offset off satisfies off + bs + 65536 >= 2^31 - 1
    uint64_t limit = 0x7FFFFFFFull - 65536ull - bs;      // off >= limit
    return (limit + bs - 1) / bs;
}

template <typename T> struct DevBuf {
    T *p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n)
    {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 8 + 256;
        cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&p), want * sizeof(T));
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

}  // namespace

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
static void pipeline_destroy(void *p);

struct lz4b200_ctx {
    void *pipe = nullptr;                     // host-batch pipeline state (streams, pinned staging), created on demand
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    uint32_t *d_tickets = nullptr;            // 3 x {next, retired}
    int dec_ctas_per_sm = 0;
    int enc16s_ctas_per_sm = 0, enc32s_ctas_per_sm = 0;   // split (matcher+emitter) encoder
    int high_priority = 0;                    // lz4b200_ctx_set_priority(ctx, 1): pipeline streams get the highest priority
    DevBuf<uint16_t> d_gtab16;                // global u16 tables (lz4_compress_blocks_gtab / _gtab16)
    const uint32_t *pipe_tickets = nullptr;  // base of the host pipeline's ticket blocks (selects a table region)
    int enc_g16 = 0;                          // LZ4B200_ENC_G16=62|71 (16-lane groups) or 862|871 (8-lane groups): lane-group matchers, 0: off
    int enc_g16_ctas = 8;                     // LZ4B200_ENC_G16_CTAS
    int enc_nib = 0;                          // (A/B build) LZ4B200_ENC_NIB=1..5: shared-memory tags + first-2 verification (gnib / gtagg)
    int enc_nib_ctas = 8;                     // LZ4B200_ENC_NIB_CTAS
    // K1-S2 (one chain per CTA over the TMA-fed ring, lz4b200_solo_kernel.cuh): LZ4B200_ENC_SOLO=2 routes batches of
    // blocks > 64 KiB (and batches of at most enc_solo_small_max small blocks) to it
    int enc_solo = 0, enc_solo_ctas_per_sm = 0, enc_solo2_ctas_per_sm = 0;
    uint32_t enc_solo_small_max = 0;
#ifdef LZ4B200_AB_VARIANTS
    int enc16_ctas_per_sm = 0, enc32_ctas_per_sm = 0;
    int enc_gtab = 71;                        // LZ4B200_ENC_GTAB=10*matchers+emitters per CTA (62|71|44|151)
    int enc_gtab_smem = 0;
    DevBuf<uint16_t> d_ttab16;                // K1-T tables
    DevBuf<uint32_t> d_gtag32;                // tagged global tables (lz4_compress_blocks_gtag)
    int enc_gtag = 0;                         // LZ4B200_ENC_GTAG=71|62: tagged entries (measured slower)
    int enc_gtag_ctas = 8;
    int enc_single_warp = 0;                  // LZ4B200_ENC_SINGLE_WARP=1: one warp searches and emits
    int dec_ctas_override = 0;                // LZ4B200_DEC_CTAS=n CTAs per SM
    int dec_conv = 0;                         // LZ4B200_DEC_CONV=1: warp-converged decoder loop
    int dec_batched = 0;                      // LZ4B200_DEC_BATCHED=1
    int dec_group_override = 0;               // LZ4B200_DEC_GROUP=4|8|16|32
    // K1-T / K2-T (one block per thread, lz4b200_thread_kernels.cuh)
    uint32_t enc_thread_min = 0xffffffffu, dec_thread_min = 0xffffffffu;
    int enc_thread_lanes = 0, dec_thread_lanes = 0;
    uint32_t enc_thread_max = 16384, dec_thread_max = 65536;
#endif
    std::string last_error;
    const char *last_kernel[2] = {"", ""};   // what the launchers picked last: [0] compress, [1] decompress (for the bench record)
    uint32_t range_nb = 0;                    // lz4b200_frame_range_compress -> _pack hand-over
    const uint8_t *range_in = nullptr;
    size_t frame_budget = 256u << 20;         // device bytes the frame decoder's block slots / staged input may take per group

    // scratch for host-pointer and frame entry points
    DevBuf<uint8_t> d_in, d_out, d_slots, d_flags, d_pick, d_dict;
    DevBuf<uint64_t> d_in_off, d_out_off, d_seg_off, d_expected, d_off_b;
    DevBuf<uint32_t> d_in_len, d_out_cap, d_out_len, d_info, d_seg_size, d_payload_len, d_link_first, d_stored_len, d_done;
    DevBuf<uint64_t> d_stored_off;
    DevBuf<int32_t> d_status;

    bool check(cudaError_t e, const char *what)
    {
        if (e == cudaSuccess) return true;
        last_error = std::string(what) + ": " + cudaGetErrorString(e);
        return false;
    }
};

namespace {

#ifdef LZ4B200_AB_VARIANTS
constexpr int kEnc16Warps = 4;     // v1 encoder: 8 KiB table per warp
constexpr int kEnc32Warps = 2;     // 2 x 16 KiB tables per CTA
#endif
#ifndef ENC16_PAIRS
#define ENC16_PAIRS 3
#endif
// Global-table encoder CTAs per SM (7 matchers + 1 emitter each, 8 KiB of table per matcher).  On an H100 the tables
// must share a 50 MB L2 with the streaming input and output: 3 CTAs (21 chains per SM, 23 MB of tables) with the register
// budget of 3 CTAs (no spills) compress 1 GiB of 64 KiB JSON blocks 2.2x faster than filling all 64 warp slots with
// 8 CTAs at 32 registers (61 MB of tables); 2, 4, 5 and 6 CTAs are slower too (DESIGN.md §6).
#ifndef ENC_GTAB_CTAS
#define ENC_GTAB_CTAS 3
#endif
constexpr int kGtabCtasPerSm = ENC_GTAB_CTAS;
#define LZ4B200_STR2(x) #x
#define LZ4B200_STR(x) LZ4B200_STR2(x)
constexpr const char *kGtabKernelName = "lz4_compress_blocks_gtab<unsigned short, 7, 1, 0, " LZ4B200_STR(ENC_GTAB_CTAS) ">";
constexpr int kEnc16Pairs = ENC16_PAIRS;   // split encoder: matcher+emitter pairs per CTA (named barriers: <= 3)
constexpr int kEnc32Pairs = 2;

#define CTX_CUDA(ctx, call)                                              \
    do {                                                                 \
        if (!(ctx)->check((call), #call)) return LZ4B200_CUDA_ERROR;     \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
    ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

template <int G>
lz4b200_status launch_decompress_g(lz4b200_ctx *ctx, const BatchArgs &a, cudaStream_t s)
{
    const uint32_t per_cta = kDecWarpsPerCta * (32 / G);
    uint32_t want = (a.nblocks + per_cta - 1) / per_cta;
    uint32_t grid = std::min<uint32_t>(want, (uint32_t)(ctx->sm_count * std::min(32, 64 / kDecWarpsPerCta)));   // 64 warps per SM
#ifdef LZ4B200_AB_VARIANTS
    if (ctx->dec_ctas_override) grid = std::min<uint32_t>(want, (uint32_t)(ctx->sm_count * ctx->dec_ctas_override));
    if (!a.dict_len && ctx->dec_conv) { lz4_decompress_blocks_conv<G><<<grid, kDecWarpsPerCta * 32, 0, s>>>(a); CTX_CUDA(ctx, cudaGetLastError()); return LZ4B200_OK; }
    if (!a.dict_len && ctx->dec_batched) { lz4_decompress_blocks<G, 1, false><<<grid, kDecWarpsPerCta * 32, 0, s>>>(a); CTX_CUDA(ctx, cudaGetLastError()); return LZ4B200_OK; }
#endif
    const uint32_t warps = (a.nblocks + (32 / G) - 1) / (32 / G);
    const bool one_warp = !a.dict_len && kDecWarpsPerCta > 1 && warps <= (uint32_t)ctx->sm_count * 32u;   // all resident as one-warp CTAs
    if (one_warp) lz4_decompress_blocks<G, 0, false, 1><<<warps, 32, 0, s>>>(a);
    else if (a.dict_len) lz4_decompress_blocks<G, 0, true><<<grid, kDecWarpsPerCta * 32, 0, s>>>(a);
    else lz4_decompress_blocks<G, 0, false><<<grid, kDecWarpsPerCta * 32, 0, s>>>(a);
    ctx->last_kernel[1] = one_warp ? (G == 8 ? "lz4_decompress_blocks<8, 0, 0, 1>" : G == 16 ? "lz4_decompress_blocks<16, 0, 0, 1>" : "lz4_decompress_blocks<32, 0, 0, 1>")
                                   : (G == 8 ? "lz4_decompress_blocks<8, 0, 0, 4>" : G == 16 ? "lz4_decompress_blocks<16, 0, 0, 4>" : "lz4_decompress_blocks<32, 0, 0, 4>");
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}

// Lanes per block: with few blocks every block gets a whole warp (widest copies, most parallel
// chains); with many blocks narrower groups cut the warp-instructions per sequence.
int pick_dec_group(const lz4b200_ctx *ctx, uint32_t nblocks)
{
#ifdef LZ4B200_AB_VARIANTS
    if (ctx->dec_group_override) return ctx->dec_group_override;
#endif
    (void)ctx;
    // narrower groups win on large batches of 64 KiB JSON blocks (fewer warp-instructions per sequence); whole warps win
    // when there are too few blocks to fill the GPU
    if (nblocks >= 12288) return 8;
    return nblocks >= 4096 ? 16 : 32;
}

#ifdef LZ4B200_AB_VARIANTS
// Active lanes per warp for the thread-per-block kernels: a batch with fewer blocks than the GPU has lanes is
// spread over more warps.
int pick_thread_lanes(const lz4b200_ctx *ctx, uint32_t threads, int override_lanes)
{
    if (override_lanes == 8 || override_lanes == 16 || override_lanes == 32) return override_lanes;
    const uint32_t full = (uint32_t)ctx->sm_count * 64u * 32u;      // every lane of every resident warp
    if (threads * 4u <= full) return 8;
    return threads * 2u <= full ? 16 : 32;
}

template <int kLanes>
lz4b200_status launch_decompress_thread(lz4b200_ctx *ctx, const BatchArgs &a, uint32_t threads, cudaStream_t s)
{
    const uint32_t per_cta = kThreadCtaWarps * kLanes;
    lz4_decompress_blocks_thread<kLanes><<<(threads + per_cta - 1) / per_cta, kThreadCtaWarps * 32, 0, s>>>(a);
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}
#endif

lz4b200_status launch_decompress(lz4b200_ctx *ctx, const BatchArgs &args, cudaStream_t s, uint32_t *tickets = nullptr)
{
    if (args.nblocks == 0) return LZ4B200_OK;
    BatchArgs a = args;
    a.tickets = tickets ? tickets : ctx->d_tickets;
#ifdef LZ4B200_AB_VARIANTS
    if (!a.dict_len && a.nblocks >= ctx->dec_thread_min) {
        const uint32_t threads = std::min(a.nblocks, ctx->dec_thread_max);
        switch (pick_thread_lanes(ctx, threads, ctx->dec_thread_lanes)) {
        case 8: return launch_decompress_thread<8>(ctx, a, threads, s);
        case 16: return launch_decompress_thread<16>(ctx, a, threads, s);
        default: return launch_decompress_thread<32>(ctx, a, threads, s);
        }
    }
    if (pick_dec_group(ctx, a.nblocks) == 4) return launch_decompress_g<4>(ctx, a, s);
#endif
    switch (pick_dec_group(ctx, a.nblocks)) {
    case 8: return launch_decompress_g<8>(ctx, a, s);
    case 16: return launch_decompress_g<16>(ctx, a, s);
    default: return launch_decompress_g<32>(ctx, a, s);
    }
}

// One table region per concurrently running launch (the host pipeline launches from up to 8 lanes): the ticket block
// doubles as the region selector.
static size_t table_slot(const lz4b200_ctx *ctx, const uint32_t *tickets)
{
    return tickets == ctx->d_tickets ? 0 : 1 + ((size_t)(tickets - ctx->pipe_tickets) / 8u) % 8u;
}

#ifdef LZ4B200_AB_VARIANTS
// The measured-and-rejected K1 variants (DESIGN.md §6).  Returns true when one of them took the batch.
static bool launch_compress_variant(lz4b200_ctx *ctx, const BatchArgs &a, uint32_t max_in_len, cudaStream_t s, uint32_t *tickets,
                                    lz4b200_status *st)
{
    *st = LZ4B200_OK;
    if (a.dict_len) return false;
    if (ctx->enc_solo == 1 && max_in_len != 0 && (max_in_len > 65536u || a.nblocks <= ctx->enc_solo_small_max)) {
        const uint32_t grid = std::min<uint32_t>(a.nblocks, (uint32_t)(ctx->sm_count * ctx->enc_solo_ctas_per_sm));
        lz4_compress_blocks_solo<<<grid, 64, kSoloSmemBytes, s>>>(a, tickets + 4);
        if (!ctx->check(cudaGetLastError(), "solo launch")) *st = LZ4B200_CUDA_ERROR;
        return true;
    }
    if (max_in_len != 0 && max_in_len <= 65536u && a.nblocks >= ctx->enc_thread_min) {
        // K1-T: one block per thread, 8 KiB table per thread in global memory
        const uint32_t threads = std::min(a.nblocks, ctx->enc_thread_max);
        const size_t region = (size_t)ctx->enc_thread_max * 4096u;                  // u16 entries
        const size_t slot = table_slot(ctx, tickets);
        if (!ctx->check(ctx->d_ttab16.reserve(region * (slot ? 9u : 1u)), "thread tables")) { *st = LZ4B200_CUDA_ERROR; return true; }
        uint16_t *gt = ctx->d_ttab16.p + slot * region;
        const int lanes = pick_thread_lanes(ctx, threads, ctx->enc_thread_lanes);
        const uint32_t per_cta = kThreadCtaWarps * lanes, grid = (threads + per_cta - 1) / per_cta;
        if (lanes == 8) lz4_compress_blocks_thread<8><<<grid, kThreadCtaWarps * 32, 0, s>>>(a, tickets + 2, gt);
        else if (lanes == 16) lz4_compress_blocks_thread<16><<<grid, kThreadCtaWarps * 32, 0, s>>>(a, tickets + 2, gt);
        else lz4_compress_blocks_thread<32><<<grid, kThreadCtaWarps * 32, 0, s>>>(a, tickets + 2, gt);
        if (!ctx->check(cudaGetLastError(), "thread launch")) *st = LZ4B200_CUDA_ERROR;
        return true;
    }
    if (max_in_len != 0 && max_in_len <= 65536u && a.nblocks > (uint32_t)ctx->sm_count * 24u) {
        const size_t slot = table_slot(ctx, tickets);
        if (ctx->enc_gtag) {                                                         // tagged (tag, position) entries
            const int m = ctx->enc_gtag / 10;
            const uint32_t grid = std::min<uint32_t>((a.nblocks + m - 1) / m, (uint32_t)(ctx->sm_count * ctx->enc_gtag_ctas));
            const size_t region = (size_t)ctx->sm_count * 8u * 8u * 4096u;
            if (!ctx->check(ctx->d_gtag32.reserve(region * 9u), "gtag")) { *st = LZ4B200_CUDA_ERROR; return true; }
            uint32_t *gt = ctx->d_gtag32.p + slot * region;
            if (m == 6) lz4_compress_blocks_gtag<6, 2><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
            else lz4_compress_blocks_gtag<7, 1><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
            if (!ctx->check(cudaGetLastError(), "gtag launch")) *st = LZ4B200_CUDA_ERROR;
            return true;
        }
        const int m = ctx->enc_gtab / 10, e = ctx->enc_gtab % 10, ks = ctx->enc_gtab_smem;
        if (ctx->enc_gtab && (m != 7 || e != 1 || ks)) {                              // other global-table CTA shapes
            const uint32_t want = (a.nblocks + m - 1) / m;
            uint32_t grid = std::min<uint32_t>(want, (uint32_t)ctx->sm_count * (m == 15 ? 4u : 8u));
            const size_t region = (size_t)ctx->sm_count * 8u * 28u * 4096u;
            if (!ctx->check(ctx->d_gtab16.reserve(region * 9u), "gtab")) { *st = LZ4B200_CUDA_ERROR; return true; }
            uint16_t *gt = ctx->d_gtab16.p + slot * region;
            if (m == 15) lz4_compress_blocks_gtab<uint16_t, 15, 1, 0><<<grid, 512, 0, s>>>(a, tickets + 2, gt);
            else if (m == 6 && e == 2) lz4_compress_blocks_gtab<uint16_t, 6, 2, 0><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
            else if (m == 4 && e == 4) lz4_compress_blocks_gtab<uint16_t, 4, 4, 0><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
            else if (ks == 2) lz4_compress_blocks_gtab<uint16_t, 7, 1, 2><<<grid, 256, 2 * 8192, s>>>(a, tickets + 2, gt);
            else if (ks == 3) {
                grid = std::min<uint32_t>(want, (uint32_t)ctx->sm_count * 7u);
                lz4_compress_blocks_gtab<uint16_t, 7, 1, 3><<<grid, 256, 3 * 8192, s>>>(a, tickets + 2, gt);
            } else return false;
            if (!ctx->check(cudaGetLastError(), "gtab launch")) *st = LZ4B200_CUDA_ERROR;
            return true;
        }
    }
    if (ctx->enc_single_warp) {                                                      // v1: one warp searches and emits
        if (max_in_len == 0 || max_in_len <= 65536u) {
            const uint32_t grid = std::min<uint32_t>((a.nblocks + kEnc16Warps - 1) / kEnc16Warps, (uint32_t)ctx->sm_count * (uint32_t)ctx->enc16_ctas_per_sm);
            lz4_compress_blocks<uint16_t, kEnc16Warps><<<grid, kEnc16Warps * 32, kEnc16Warps * 4096 * sizeof(uint16_t), s>>>(a, tickets + 2);
        }
        if (max_in_len == 0 || max_in_len > 65536u) {
            const uint32_t grid = std::min<uint32_t>((a.nblocks + kEnc32Warps - 1) / kEnc32Warps, (uint32_t)(ctx->sm_count * ctx->enc32_ctas_per_sm));
            lz4_compress_blocks<uint32_t, kEnc32Warps><<<grid, kEnc32Warps * 32, kEnc32Warps * 4096 * sizeof(uint32_t), s>>>(a, tickets + 4);
        }
        if (!ctx->check(cudaGetLastError(), "v1 launch")) *st = LZ4B200_CUDA_ERROR;
        return true;
    }
    return false;
}
#endif

// K1 launcher.  Blocks <= 64 KiB: u16 tables; larger: u32 tables; unknown mix (max_in_len == 0): both kernels run over
// the same ticket space and each skips the other's blocks.
//   many small blocks (> 24 per SM, no dictionary)  -> global tables (21 chains per SM; lane-group matchers: more)
//   fewer / dictionary                              -> shared-memory tables, matcher + emitter pairs
//   blocks > 64 KiB without dictionary              -> one chain per CTA over the TMA-fed ring when enabled
lz4b200_status launch_compress(lz4b200_ctx *ctx, const BatchArgs &args, uint32_t max_in_len, cudaStream_t s,
                               uint32_t *tickets = nullptr)
{
    if (!tickets) tickets = ctx->d_tickets;
    if (args.nblocks == 0) return LZ4B200_OK;
    const BatchArgs &a = args;
#ifdef LZ4B200_AB_VARIANTS
    {
        lz4b200_status vst;
        if (launch_compress_variant(ctx, a, max_in_len, s, tickets, &vst)) return vst;
    }
#endif
    if (!a.dict_len && ctx->enc_solo == 2 && max_in_len != 0 && (max_in_len > 65536u || a.nblocks <= ctx->enc_solo_small_max)) {
        const uint32_t grid = std::min<uint32_t>(a.nblocks, (uint32_t)(ctx->sm_count * ctx->enc_solo2_ctas_per_sm));
        lz4_compress_blocks_solo2<<<grid, 64, kSolo2SmemBytes, s>>>(a, tickets + 4);
        ctx->last_kernel[0] = "lz4_compress_blocks_solo2";
        CTX_CUDA(ctx, cudaGetLastError());
        return LZ4B200_OK;
    }
    {                                                       // u16 tables: every block with input (+ dictionary) <= 64 KiB
        if (!a.dict_len && a.nblocks > (uint32_t)ctx->sm_count * 24u) {
            // u16 entries: CTAs per SM x chains per CTA tables of 4096, one region per concurrently running launch
            const int g16_m = (ctx->enc_g16 % 100) / 10, g16_g = ctx->enc_g16 >= 800 ? 8 : 16;
            const size_t chains_per_sm = ctx->enc_g16 ? (size_t)ctx->enc_g16_ctas * (32 / g16_g) * g16_m : (ctx->enc_nib >= 4 ? 112u : ctx->enc_nib ? 8u * 7u : (size_t)kGtabCtasPerSm * 7u);   // enc_nib: A/B build only
            const size_t region = (size_t)ctx->sm_count * chains_per_sm * 4096u;
            if (!ctx->check(ctx->d_gtab16.reserve(region * 9u), "gtab")) return LZ4B200_CUDA_ERROR;
            uint16_t *gt = ctx->d_gtab16.p + table_slot(ctx, tickets) * region;
#ifdef LZ4B200_AB_VARIANTS
            if (ctx->enc_nib && !ctx->enc_g16) {                                     // tags in shared memory: 1 = nibbles x 8 CTAs, 2 = bytes x 6 CTAs, 3 = nibbles x 6 CTAs (40 registers)
                const uint32_t ctas = std::min(ctx->enc_nib_ctas, ctx->enc_nib == 1 ? 8 : 6);
                const uint32_t grid = std::min<uint32_t>((a.nblocks + 6) / 7, (uint32_t)ctx->sm_count * ctas);
                if (ctx->enc_nib == 4) {                                             // lane groups of 8 + 2-bit tags: 4 x 28 chains per SM
                    const uint32_t g4 = std::min<uint32_t>((a.nblocks + 27) / 28, (uint32_t)ctx->sm_count * std::min(ctx->enc_nib_ctas, 4));
                    lz4_compress_blocks_gtagg<8, 7, 1, 2, 4><<<g4, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtagg<8, 7, 1, 2, 4>";
                } else if (ctx->enc_nib == 5) {                                      // lane groups of 16 + 2-bit tags: 8 x 14 chains per SM
                    const uint32_t g5 = std::min<uint32_t>((a.nblocks + 13) / 14, (uint32_t)ctx->sm_count * std::min(ctx->enc_nib_ctas, 8));
                    lz4_compress_blocks_gtagg<16, 7, 1, 2, 8><<<g5, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtagg<16, 7, 1, 2, 8>";
                } else
                if (ctx->enc_nib == 2) { lz4_compress_blocks_gnib<7, 1, 8, 6><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gnib<7, 1, 8, 6>"; }
                else if (ctx->enc_nib == 3) { lz4_compress_blocks_gnib<7, 1, 4, 6><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gnib<7, 1, 4, 6>"; }
                else { lz4_compress_blocks_gnib<7, 1, 4, 8><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gnib<7, 1, 4, 8>"; }
            } else
#endif
            if (ctx->enc_g16) {                                               // 2 or 4 chains per matcher warp
                const int m = (ctx->enc_g16 % 100) / 10, gsz = ctx->enc_g16 >= 800 ? 8 : 16;   // 62 | 71 (G = 16), 862 | 871 (G = 8)
                const int per_cta = (32 / gsz) * m;
                const uint32_t grid = std::min<uint32_t>((a.nblocks + per_cta - 1) / per_cta, (uint32_t)(ctx->sm_count * ctx->enc_g16_ctas));
                if (gsz == 8 && m == 7) { lz4_compress_blocks_gtabg<8, 7, 1><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtabg<8, 7, 1>"; }
                else if (gsz == 8) { lz4_compress_blocks_gtabg<8, 6, 2><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtabg<8, 6, 2>"; }
                else if (m == 7) { lz4_compress_blocks_gtabg<16, 7, 1><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtabg<16, 7, 1>"; }
                else { lz4_compress_blocks_gtabg<16, 6, 2><<<grid, 256, 0, s>>>(a, tickets + 2, gt); ctx->last_kernel[0] = "lz4_compress_blocks_gtabg<16, 6, 2>"; }
            } else {
                const uint32_t grid = std::min<uint32_t>((a.nblocks + 6) / 7, (uint32_t)ctx->sm_count * kGtabCtasPerSm);
                lz4_compress_blocks_gtab<uint16_t, 7, 1, 0, kGtabCtasPerSm><<<grid, 256, 0, s>>>(a, tickets + 2, gt);
                ctx->last_kernel[0] = kGtabKernelName;
            }
        } else {
            ctx->last_kernel[0] = "lz4_compress_blocks_split<unsigned short, 3, 0>";
            const uint32_t grid = std::min<uint32_t>((a.nblocks + kEnc16Pairs - 1) / kEnc16Pairs, (uint32_t)(ctx->sm_count * ctx->enc16s_ctas_per_sm));
            if (a.dict_len)
                lz4_compress_blocks_split<uint16_t, kEnc16Pairs, true>
                    <<<grid, kEnc16Pairs * 64, split_smem_bytes<uint16_t, kEnc16Pairs>(), s>>>(a, tickets + 2);
            else
                lz4_compress_blocks_split<uint16_t, kEnc16Pairs, false>
                    <<<grid, kEnc16Pairs * 64, split_smem_bytes<uint16_t, kEnc16Pairs>(), s>>>(a, tickets + 2);
        }
        CTX_CUDA(ctx, cudaGetLastError());
    }
    if (max_in_len == 0 || (uint64_t)max_in_len + a.dict_len > 65536u) {
        if (max_in_len > 65536u) ctx->last_kernel[0] = "lz4_compress_blocks_split<unsigned int, 2, 0>";
        const uint32_t grid = std::min<uint32_t>((a.nblocks + kEnc32Pairs - 1) / kEnc32Pairs, (uint32_t)(ctx->sm_count * ctx->enc32s_ctas_per_sm));
        if (a.dict_len)
            lz4_compress_blocks_split<uint32_t, kEnc32Pairs, true>
                <<<grid, kEnc32Pairs * 64, split_smem_bytes<uint32_t, kEnc32Pairs>(), s>>>(a, tickets + 4);
        else
            lz4_compress_blocks_split<uint32_t, kEnc32Pairs, false>
                <<<grid, kEnc32Pairs * 64, split_smem_bytes<uint32_t, kEnc32Pairs>(), s>>>(a, tickets + 4);
        CTX_CUDA(ctx, cudaGetLastError());
    }
    return LZ4B200_OK;
}

}  // namespace

extern "C" {

int lz4b200_abi_version(void) { return LZ4B200_ABI_VERSION; }

int lz4b200_host_pointer_kind(const void *p)
{
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return -1; }
    return (int)a.type;                       // 0 unregistered (pageable), 1 host (pinned), 2 device, 3 managed
}

const char *lz4b200_status_string(int s)
{
    switch (s) {
    case LZ4B200_OK: return "ok";
    case LZ4B200_COMPRESS_OUTPUT_TOO_SMALL:
        return "output is too small for the compressed data, use get_maximum_output_size to reserve enough space";
    case LZ4B200_DEC_OUTPUT_TOO_SMALL: return "provided output is too small for the decompressed data";
    case LZ4B200_DEC_LITERAL_OUT_OF_BOUNDS: return "literal is out of bounds of the input";
    case LZ4B200_DEC_EXPECTED_ANOTHER_BYTE: return "expected another byte, found none";
    case LZ4B200_DEC_OFFSET_ZERO: return "0 is not a valid match offset";
    case LZ4B200_DEC_OFFSET_OUT_OF_BOUNDS: return "the offset to copy is not contained in the decompressed buffer";
    case LZ4B200_FRAME_DECOMPRESSION_ERROR: return "frame: block decompression error";
    case LZ4B200_FRAME_WRONG_MAGIC: return "frame: wrong magic number";
    case LZ4B200_FRAME_RESERVED_BITS: return "frame: reserved bits set";
    case LZ4B200_FRAME_UNSUPPORTED_VERSION: return "frame: unsupported version";
    case LZ4B200_FRAME_UNSUPPORTED_BLOCKSIZE: return "frame: unsupported block size";
    case LZ4B200_FRAME_HEADER_CHECKSUM: return "frame: header checksum error";
    case LZ4B200_FRAME_BLOCK_CHECKSUM: return "frame: block checksum error";
    case LZ4B200_FRAME_CONTENT_CHECKSUM: return "frame: content checksum error";
    case LZ4B200_FRAME_CONTENT_LENGTH: return "frame: content length differs from the header";
    case LZ4B200_FRAME_BLOCK_TOO_BIG: return "frame: block too big";
    case LZ4B200_FRAME_SKIPPABLE: return "frame: skippable frame";
    case LZ4B200_FRAME_DICTIONARY: return "frame: dictionaries are not supported";
    case LZ4B200_FRAME_IO_EOF: return "frame: unexpected end of input";
    case LZ4B200_FRAME_LINKED_UNSUPPORTED: return "frame: linked blocks are not supported on the GPU path";
    case LZ4B200_FRAME_OUTPUT_FULL: return "frame: output buffer exhausted";
    case LZ4B200_INVALID_ARGUMENT: return "invalid argument";
    case LZ4B200_CUDA_ERROR: return "CUDA error";
    default: return "unknown status";
    }
}

const char *lz4b200_last_cuda_error(const lz4b200_ctx *ctx) { return ctx ? ctx->last_error.c_str() : ""; }

lz4b200_status lz4b200_ctx_create(int device, lz4b200_ctx **out)
{
    if (!out) return LZ4B200_INVALID_ARGUMENT;
    *out = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) return LZ4B200_CUDA_ERROR;
    lz4b200_ctx *ctx = new lz4b200_ctx();
    ctx->device = device;
    DeviceGuard guard(device);
    bool ok = ctx->check(cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device), "sm count") &&
              ctx->check(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking), "stream") &&
              ctx->check(cudaMalloc(reinterpret_cast<void **>(&ctx->d_tickets), 8 * sizeof(uint32_t)), "tickets") &&
              ctx->check(cudaMemset(ctx->d_tickets, 0, 8 * sizeof(uint32_t)), "tickets memset");
    if (ok) {
        ok = ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->dec_ctas_per_sm, lz4_decompress_blocks<8, 0, false>,
                                                                      kDecWarpsPerCta * 32, 0), "occupancy dec") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                            &ctx->enc16s_ctas_per_sm, lz4_compress_blocks_split<uint16_t, kEnc16Pairs, false>, kEnc16Pairs * 64,
                            split_smem_bytes<uint16_t, kEnc16Pairs>()), "occupancy enc16 split") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                            &ctx->enc32s_ctas_per_sm, lz4_compress_blocks_split<uint32_t, kEnc32Pairs, false>, kEnc32Pairs * 64,
                            split_smem_bytes<uint32_t, kEnc32Pairs>()), "occupancy enc32 split") &&
             ctx->check(cudaFuncSetAttribute(lz4_compress_blocks_solo2, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)kSolo2SmemBytes), "solo2 smem") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->enc_solo2_ctas_per_sm, lz4_compress_blocks_solo2, 64,
                                                                      kSolo2SmemBytes), "occupancy solo2");
        ctx->enc_solo_small_max = (uint32_t)(ctx->sm_count * std::max(1, ctx->enc_solo2_ctas_per_sm));
    }
#ifdef LZ4B200_AB_VARIANTS
    if (ok) {
        ok = ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                            &ctx->enc16_ctas_per_sm, lz4_compress_blocks<uint16_t, kEnc16Warps>, kEnc16Warps * 32,
                            kEnc16Warps * 4096 * sizeof(uint16_t)), "occupancy enc16") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(
                            &ctx->enc32_ctas_per_sm, lz4_compress_blocks<uint32_t, kEnc32Warps>, kEnc32Warps * 32,
                            kEnc32Warps * 4096 * sizeof(uint32_t)), "occupancy enc32") &&
             ctx->check(cudaFuncSetAttribute(lz4_compress_blocks_solo, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             (int)kSoloSmemBytes), "solo smem") &&
             ctx->check(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&ctx->enc_solo_ctas_per_sm, lz4_compress_blocks_solo, 64,
                                                                      kSoloSmemBytes), "occupancy solo");
    }
#endif
    if (!ok || ctx->dec_ctas_per_sm < 1 || ctx->enc16s_ctas_per_sm < 1 || ctx->enc32s_ctas_per_sm < 1) {
        fprintf(stderr, "lz4b200: context creation failed: %s\n", ctx->last_error.c_str());
        lz4b200_ctx_destroy(ctx);
        return LZ4B200_CUDA_ERROR;
    }
    // The global-table encoders mark their table accesses L2::evict_last; how much of the L2 such lines may occupy is the
    // device's persisting-L2 limit (LZ4B200_L2_PERSIST_MB sets it; unset = leave the process's setting alone).
    if (const char *g = getenv("LZ4B200_L2_PERSIST_MB")) {
        int maxp = 0;
        cudaDeviceGetAttribute(&maxp, cudaDevAttrMaxPersistingL2CacheSize, device);
        const size_t bytes = std::min<size_t>((size_t)std::max(0L, atol(g)) << 20, (size_t)maxp);
        const cudaError_t e = cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, bytes);
        if (getenv("LZ4B200_DEBUG"))
            fprintf(stderr, "lz4b200: persisting L2 limit %zu of max %d bytes: %s\n", bytes, maxp, cudaGetErrorString(e));
    }
    if (const char *g = getenv("LZ4B200_ENC_G16")) ctx->enc_g16 = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_G16_CTAS")) ctx->enc_g16_ctas = std::max(1, std::min(8, atoi(g)));
#ifdef LZ4B200_AB_VARIANTS
    if (const char *g = getenv("LZ4B200_ENC_NIB")) ctx->enc_nib = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_NIB_CTAS")) ctx->enc_nib_ctas = std::max(1, std::min(8, atoi(g)));
#endif
    if (const char *g = getenv("LZ4B200_ENC_SOLO")) ctx->enc_solo = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_SOLO_SMALL_MAX")) ctx->enc_solo_small_max = (uint32_t)atoll(g);
    if (ctx->enc_solo2_ctas_per_sm < 1 && ctx->enc_solo == 2) ctx->enc_solo = 0;
    if (getenv("LZ4B200_DEBUG"))
        fprintf(stderr, "lz4b200: SMs %d, CTAs/SM: dec %d, enc16-split %d (x%d pairs), enc32-split %d (x%d pairs), solo2 %d\n",
                ctx->sm_count, ctx->dec_ctas_per_sm, ctx->enc16s_ctas_per_sm, kEnc16Pairs, ctx->enc32s_ctas_per_sm, kEnc32Pairs,
                ctx->enc_solo2_ctas_per_sm);
#ifdef LZ4B200_AB_VARIANTS
    if (ctx->enc_solo == 1 && ctx->enc_solo_ctas_per_sm < 1) ctx->enc_solo = 0;
    if (const char *g = getenv("LZ4B200_ENC_SINGLE_WARP")) ctx->enc_single_warp = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_GTAB")) ctx->enc_gtab = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_GTAG")) ctx->enc_gtag = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_GTAG_CTAS")) ctx->enc_gtag_ctas = std::max(1, std::min(8, atoi(g)));
    if (const char *g = getenv("LZ4B200_ENC_GTAB_SMEM")) ctx->enc_gtab_smem = atoi(g);
    if (const char *g = getenv("LZ4B200_DEC_CTAS")) ctx->dec_ctas_override = atoi(g);
    if (const char *g = getenv("LZ4B200_DEC_BATCHED")) ctx->dec_batched = atoi(g);
    if (const char *g = getenv("LZ4B200_DEC_CONV")) ctx->dec_conv = atoi(g);
    if (const char *g = getenv("LZ4B200_THREAD_MIN")) ctx->enc_thread_min = ctx->dec_thread_min = (uint32_t)atoll(g);
    if (const char *g = getenv("LZ4B200_ENC_THREAD_MIN")) ctx->enc_thread_min = (uint32_t)atoll(g);
    if (const char *g = getenv("LZ4B200_DEC_THREAD_MIN")) ctx->dec_thread_min = (uint32_t)atoll(g);
    if (const char *g = getenv("LZ4B200_ENC_THREAD_LANES")) ctx->enc_thread_lanes = atoi(g);
    if (const char *g = getenv("LZ4B200_DEC_THREAD_LANES")) ctx->dec_thread_lanes = atoi(g);
    if (const char *g = getenv("LZ4B200_ENC_THREADS")) ctx->enc_thread_max = std::max(32, atoi(g));
    if (const char *g = getenv("LZ4B200_DEC_THREADS")) ctx->dec_thread_max = std::max(32, atoi(g));
    if (const char *g = getenv("LZ4B200_DEC_GROUP")) {
        int v = atoi(g);
        if (v == 4 || v == 8 || v == 16 || v == 32) ctx->dec_group_override = v;
    }
#else
    if (ctx->enc_solo == 1) ctx->enc_solo = 0;               // the single-thread solo kernel only exists in the A/B build
#endif
    *out = ctx;
    return LZ4B200_OK;
}

void lz4b200_ctx_destroy(lz4b200_ctx *ctx)
{
    if (!ctx) return;
    DeviceGuard guard(ctx->device);
    if (ctx->stream) { cudaStreamSynchronize(ctx->stream); cudaStreamDestroy(ctx->stream); }
    if (ctx->d_tickets) cudaFree(ctx->d_tickets);
    pipeline_destroy(ctx->pipe);
    ctx->d_in.release(); ctx->d_out.release(); ctx->d_slots.release(); ctx->d_flags.release(); ctx->d_pick.release();
    ctx->d_in_off.release(); ctx->d_out_off.release(); ctx->d_seg_off.release(); ctx->d_expected.release();
    ctx->d_off_b.release();
    ctx->d_in_len.release(); ctx->d_out_cap.release(); ctx->d_out_len.release(); ctx->d_info.release();
    ctx->d_seg_size.release(); ctx->d_payload_len.release(); ctx->d_status.release();
    ctx->d_gtab16.release();
#ifdef LZ4B200_AB_VARIANTS
    ctx->d_ttab16.release(); ctx->d_gtag32.release();
#endif
    delete ctx;
}

void lz4b200_ctx_set_priority(lz4b200_ctx *ctx, int high)
{
    if (ctx && !ctx->pipe) ctx->high_priority = high != 0;    // takes effect when the pipeline streams are created
}

void *lz4b200_ctx_stream(lz4b200_ctx *ctx) { return ctx ? (void *)ctx->stream : nullptr; }

const char *lz4b200_ctx_last_kernel(const lz4b200_ctx *ctx, int which)
{
    return ctx && (which == 0 || which == 1) ? ctx->last_kernel[which] : "";
}

size_t lz4b200_max_output_size(size_t n) { return 16 + 4 + (size_t)((uint64_t)n * 110 / 100); }

uint32_t lz4b200_xxh32(const uint8_t *data, size_t n, uint32_t seed)
{
    Xxh32 h(seed);
    h.update(data, n);
    return h.digest();
}

void lz4b200_xxh32_reset(lz4b200_xxh32_state *st, uint32_t seed)
{
    Xxh32 h(seed);
    memcpy(st->acc, h.acc, sizeof st->acc);
    st->fill = 0; st->seed = seed; st->total = 0;
}

void lz4b200_xxh32_update(lz4b200_xxh32_state *st, const uint8_t *data, size_t n)
{
    Xxh32 h(st->seed);
    memcpy(h.acc, st->acc, sizeof st->acc); memcpy(h.buf, st->buf, 16); h.fill = st->fill; h.total = st->total;
    h.update(data, n);
    memcpy(st->acc, h.acc, sizeof st->acc); memcpy(st->buf, h.buf, 16); st->fill = h.fill; st->total = h.total;
}

uint32_t lz4b200_xxh32_digest(const lz4b200_xxh32_state *st)
{
    Xxh32 h(st->seed);
    memcpy(h.acc, st->acc, sizeof st->acc); memcpy(h.buf, st->buf, 16); h.fill = st->fill; h.total = st->total;
    return h.digest();
}

// ---- device batch entry points ----------------------------------------------------------------

lz4b200_status lz4b200_compress_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                                             const uint32_t *d_in_len, const uint8_t *d_flags, uint8_t *d_out,
                                             const uint64_t *d_out_off, const uint32_t *d_out_cap,
                                             uint32_t *d_out_len, int32_t *d_status, size_t nblocks,
                                             uint32_t max_in_len, void *stream)
{
    if (!ctx || nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_out || !d_out_off || !d_out_cap || !d_out_len || !d_status))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    BatchArgs a{d_in, d_in_off, d_in_len, d_flags, d_out, d_out_off, d_out_cap, d_out_len, d_status, nullptr,
                (uint32_t)nblocks, nullptr};
    return launch_compress(ctx, a, max_in_len, (cudaStream_t)stream);
}

lz4b200_status lz4b200_decompress_batch_device(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                                               const uint32_t *d_in_len, uint8_t *d_out, const uint64_t *d_out_off,
                                               const uint32_t *d_out_cap, uint32_t *d_out_len, int32_t *d_status,
                                               uint64_t *d_err_expected, size_t nblocks, void *stream)
{
    if (!ctx || nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_out || !d_out_off || !d_out_cap || !d_out_len || !d_status))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    BatchArgs a{d_in, d_in_off, d_in_len, nullptr, d_out, d_out_off, d_out_cap, d_out_len, d_status, d_err_expected,
                (uint32_t)nblocks, nullptr};
    return launch_decompress(ctx, a, (cudaStream_t)stream);
}

// Device-pointer batches with an external dictionary shared by every block (d_dict: the LAST min(len, 65536)
// bytes of the dictionary, already on the device; compress drops dictionaries of <= 3 bytes like the reference).
lz4b200_status lz4b200_compress_batch_device_with_dict(lz4b200_ctx *ctx, const uint8_t *d_in, const uint64_t *d_in_off,
                                                       const uint32_t *d_in_len, const uint8_t *d_dict, size_t dict_len,
                                                       uint8_t *d_out, const uint64_t *d_out_off,
                                                       const uint32_t *d_out_cap, uint32_t *d_out_len,
                                                       int32_t *d_status, size_t nblocks, uint32_t max_in_len,
                                                       void *stream)
{
    if (!ctx || nblocks > 0xffffffffull || (!d_dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_out || !d_out_off || !d_out_cap || !d_out_len || !d_status))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    BatchArgs a{d_in, d_in_off, d_in_len, nullptr, d_out, d_out_off, d_out_cap, d_out_len, d_status, nullptr,
                (uint32_t)nblocks, nullptr};
    if (dict_len > 3) {
        if (dict_len > 65536) { d_dict += dict_len - 65536; dict_len = 65536; }
        a.dict = d_dict; a.dict_len = (uint32_t)dict_len;
    }
    return launch_compress(ctx, a, max_in_len, (cudaStream_t)stream);
}

lz4b200_status lz4b200_decompress_batch_device_with_dict(lz4b200_ctx *ctx, const uint8_t *d_in,
                                                         const uint64_t *d_in_off, const uint32_t *d_in_len,
                                                         const uint8_t *d_dict, size_t dict_len, uint8_t *d_out,
                                                         const uint64_t *d_out_off, const uint32_t *d_out_cap,
                                                         uint32_t *d_out_len, int32_t *d_status,
                                                         uint64_t *d_err_expected, size_t nblocks, void *stream)
{
    if (!ctx || nblocks > 0xffffffffull || (!d_dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks && (!d_in || !d_in_off || !d_in_len || !d_out || !d_out_off || !d_out_cap || !d_out_len || !d_status))
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    BatchArgs a{d_in, d_in_off, d_in_len, nullptr, d_out, d_out_off, d_out_cap, d_out_len, d_status, d_err_expected,
                (uint32_t)nblocks, nullptr};
    if (dict_len) {
        if (dict_len > 65536) { d_dict += dict_len - 65536; dict_len = 65536; }
        a.dict = d_dict; a.dict_len = (uint32_t)dict_len;
    }
    return launch_decompress(ctx, a, (cudaStream_t)stream);
}

// ---- host batch entry points --------------------------------------------------------------------
// Both calls are chunked software pipelines over kLanes streams: while chunk c runs its kernel, chunk
// c+1's input crosses PCIe host->device and chunk c-1's result crosses device->host (full duplex), so
// a large batch runs at max(PCIe, kernel) instead of their sum.

}  // extern "C"

namespace {

constexpr int kMaxLanes = 8;
// Lanes in flight.  A compress chunk occupies its lane for H2D + kernel (at least one block's serial chain, several ms)
// + the size read-back + D2H, so a few lanes cap the call whatever the kernel does; eight lanes leave the kernel / PCIe as
// the bound.  LZ4B200_LANES overrides.
static int lanes_in_use()
{
    static const int v = [] { const char *e = getenv("LZ4B200_LANES"); int k = e ? atoi(e) : 8; return k < 1 ? 1 : (k > kMaxLanes ? kMaxLanes : k); }();
    return v;
}
// decompress: a chunk's kernel lasts at least one block's serial chain (about a millisecond for 64 KiB of JSON) however
// few blocks it holds, so chunks must be big enough for that to hide behind the chunk's own D2H copy
constexpr uint64_t kChunkBytesDefault = 128ull << 20;
// compress: a 64 KiB block is one serial chain of several ms whatever the batch size, so a chunk must hold enough blocks
// (2048) for two chunks in flight to fill the GPU
constexpr uint64_t kCompressChunkBytesDefault = 128ull << 20;

uint64_t env_mib(const char *name, uint64_t dflt)         // tuning aid: chunk sizes in MiB
{
    const char *v = getenv(name);
    const long m = v ? atol(v) : 0;
    return m > 0 ? (uint64_t)m << 20 : dflt;
}

struct Lane {
    cudaStream_t stream = nullptr;
    cudaEvent_t sizes_ready = nullptr;
    DevBuf<uint8_t> in, slots, out;
};

struct Pipeline {
    Lane lane[kMaxLanes];
    cudaEvent_t desc_ready = nullptr;
    uint32_t *d_tickets = nullptr;           // kMaxLanes x 8 counters
    uint64_t *h_seg = nullptr; size_t h_seg_cap = 0;       // pinned
    int32_t *h_status = nullptr; size_t h_status_cap = 0;  // pinned
    bool ready = false;
};

lz4b200_status pipeline_init(lz4b200_ctx *ctx, Pipeline &p)
{
    if (p.ready) return LZ4B200_OK;
    for (int i = 0; i < kMaxLanes; i++) {
        // LZ4B200_STREAM_PRIORITY=high: this context's kernels get the SM slots first when another context (e.g. a
        // compress pipeline running next to a decompress pipeline) keeps the GPU full
        int lo = 0, hi = 0;
        cudaDeviceGetStreamPriorityRange(&lo, &hi);
        const int prio = ctx->high_priority ? hi : 0;
        CTX_CUDA(ctx, cudaStreamCreateWithPriority(&p.lane[i].stream, cudaStreamNonBlocking, prio));
        CTX_CUDA(ctx, cudaEventCreateWithFlags(&p.lane[i].sizes_ready, cudaEventDisableTiming));
    }
    CTX_CUDA(ctx, cudaEventCreateWithFlags(&p.desc_ready, cudaEventDisableTiming));
    CTX_CUDA(ctx, cudaMalloc(reinterpret_cast<void **>(&p.d_tickets), kMaxLanes * 8 * sizeof(uint32_t)));
    CTX_CUDA(ctx, cudaMemset(p.d_tickets, 0, kMaxLanes * 8 * sizeof(uint32_t)));
    ctx->pipe_tickets = p.d_tickets;
    p.ready = true;
    return LZ4B200_OK;
}

template <typename T> cudaError_t pinned_reserve(T *&ptr, size_t &cap, size_t n)
{
    if (n <= cap) return cudaSuccess;
    if (ptr) cudaFreeHost(ptr);
    ptr = nullptr; cap = 0;
    cudaError_t e = cudaHostAlloc(reinterpret_cast<void **>(&ptr), (n + n / 4 + 64) * sizeof(T), cudaHostAllocDefault);
    if (e == cudaSuccess) cap = n + n / 4 + 64;
    return e;
}

struct Chunk { uint32_t b0, b1; uint64_t in_lo, in_hi, a, b; };   // a/b: slot bytes (compress) or out_lo/out_hi (decompress)

}  // namespace

static Pipeline &ctx_pipeline(lz4b200_ctx *ctx)
{
    if (!ctx->pipe) ctx->pipe = new Pipeline();
    return *static_cast<Pipeline *>(ctx->pipe);
}

static void pipeline_destroy(void *vp)
{
    Pipeline *p = static_cast<Pipeline *>(vp);
    if (!p) return;
    for (int i = 0; i < kMaxLanes; i++) {
        if (p->lane[i].stream) { cudaStreamSynchronize(p->lane[i].stream); cudaStreamDestroy(p->lane[i].stream); }
        if (p->lane[i].sizes_ready) cudaEventDestroy(p->lane[i].sizes_ready);
        p->lane[i].in.release(); p->lane[i].slots.release(); p->lane[i].out.release();
    }
    if (p->desc_ready) cudaEventDestroy(p->desc_ready);
    if (p->d_tickets) cudaFree(p->d_tickets);
    if (p->h_seg) cudaFreeHost(p->h_seg);
    if (p->h_status) cudaFreeHost(p->h_status);
    delete p;
}

// The reference keeps only the last WINDOW_SIZE bytes of a dictionary (init_dict, compress.rs:571-575) and drops
// dictionaries of <= 3 bytes (compress_into_vec_with_dict, compress.rs:626-628).
static void normalize_dict(const uint8_t *&dict, size_t &dict_len, bool for_compress)
{
    if (!dict || (for_compress && dict_len <= 3)) { dict = nullptr; dict_len = 0; return; }
    if (dict_len > 65536) { dict += dict_len - 65536; dict_len = 65536; }
}

static lz4b200_status compress_batch_host_impl(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                               const uint32_t *in_len, const uint8_t *flags, const uint8_t *dict,
                                               size_t dict_len, uint8_t *out, size_t out_cap_total, uint64_t *out_off,
                                               uint32_t *out_len, int32_t *status, size_t nblocks)
{
    if (!ctx || nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks == 0) return LZ4B200_OK;
    if (!in || !in_off || !in_len || !out || !out_off || !out_len || !status) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    Pipeline &pl = ctx_pipeline(ctx);
    const int kLanes = lanes_in_use();
    lz4b200_status st = pipeline_init(ctx, pl);
    if (st != LZ4B200_OK) return st;
    const uint32_t nb = (uint32_t)nblocks;

    // ---- plan: chunks of ~kCompressChunkBytes input, descriptors relative to each chunk's buffers ------
    static const uint64_t kCompressChunkBytes = env_mib("LZ4B200_ENC_CHUNK_MB", kCompressChunkBytesDefault);
    std::vector<Chunk> chunks;
    std::vector<uint64_t> h_in_off(nb), h_slot_off(nb);
    std::vector<uint32_t> h_cap(nb);
    uint32_t max_len = 0;
    for (uint32_t b = 0; b < nb;) {
        Chunk c{b, b, ~0ull, 0, 0, 0};
        uint64_t bytes = 0;
        // ramp: the first chunks are small (32, 64, ... MiB) so the first kernel starts after a short copy.  (Shrinking the
        // LAST chunks as well — so that less work waits behind the last copy — was measured slower: the extra chunks'
        // read-back / pack / D2H round trips cost more than the shorter tail saves.)
        const uint64_t limit = std::min<uint64_t>(kCompressChunkBytes, (32ull << 20) << std::min<size_t>(chunks.size(), 8));
        while (c.b1 < nb && (c.b1 == c.b0 || bytes + in_len[c.b1] <= limit)) {
            const uint32_t k = c.b1++;
            c.in_lo = std::min<uint64_t>(c.in_lo, in_off[k]);
            c.in_hi = std::max<uint64_t>(c.in_hi, in_off[k] + in_len[k]);
            bytes += in_len[k];
            max_len = std::max(max_len, in_len[k]);
            const size_t m = lz4b200_max_output_size(in_len[k]);
            if (m > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
            h_cap[k] = (uint32_t)m;
            h_slot_off[k] = c.a;
            c.a += (m + 15) & ~size_t(15);
        }
        for (uint32_t k = c.b0; k < c.b1; k++) h_in_off[k] = in_off[k] - c.in_lo;
        chunks.push_back(c);
        b = c.b1;
    }
    const uint32_t nch = (uint32_t)chunks.size();
    CTX_CUDA(ctx, ctx->d_in_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_in_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_status.reserve(nb));
    CTX_CUDA(ctx, ctx->d_seg_off.reserve(nb + nch));
    if (flags) CTX_CUDA(ctx, ctx->d_flags.reserve(nb));
    CTX_CUDA(ctx, pinned_reserve(pl.h_seg, pl.h_seg_cap, (size_t)nb + nch));
    CTX_CUDA(ctx, pinned_reserve(pl.h_status, pl.h_status_cap, nb));

    cudaStream_t s0 = pl.lane[0].stream;
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_off.p, h_in_off.data(), nb * 8, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_len.p, in_len, nb * 4, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_off.p, h_slot_off.data(), nb * 8, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_cap.p, h_cap.data(), nb * 4, cudaMemcpyHostToDevice, s0));
    if (flags) CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_flags.p, flags, nb, cudaMemcpyHostToDevice, s0));
    normalize_dict(dict, dict_len, true);
    if (dict_len) {
        CTX_CUDA(ctx, ctx->d_dict.reserve(dict_len + 16));
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_dict.p, dict, dict_len, cudaMemcpyHostToDevice, s0));
    }
    CTX_CUDA(ctx, cudaEventRecord(pl.desc_ready, s0));
    CTX_CUDA(ctx, cudaStreamSynchronize(s0));            // the host vectors above may go out of scope before use otherwise

    auto phase1 = [&](uint32_t ci) -> lz4b200_status {  // H2D + kernel + scan + sizes D2H
        const Chunk &c = chunks[ci];
        Lane &ln = pl.lane[ci % kLanes];
        const uint32_t n = c.b1 - c.b0;
        CTX_CUDA(ctx, ln.in.reserve(c.in_hi - c.in_lo + 16));
        CTX_CUDA(ctx, ln.slots.reserve(c.a + 16));
        CTX_CUDA(ctx, cudaStreamWaitEvent(ln.stream, pl.desc_ready, 0));
        CTX_CUDA(ctx, cudaMemcpyAsync(ln.in.p, in + c.in_lo, c.in_hi - c.in_lo, cudaMemcpyHostToDevice, ln.stream));
        BatchArgs a{ln.in.p, ctx->d_in_off.p + c.b0, ctx->d_in_len.p + c.b0, flags ? ctx->d_flags.p + c.b0 : nullptr,
                    ln.slots.p, ctx->d_out_off.p + c.b0, ctx->d_out_cap.p + c.b0, ctx->d_out_len.p + c.b0,
                    ctx->d_status.p + c.b0, nullptr, n, nullptr};
        if (dict_len) { a.dict = ctx->d_dict.p; a.dict_len = (uint32_t)dict_len; }
        lz4b200_status r = launch_compress(ctx, a, max_len, ln.stream, pl.d_tickets + 8 * (ci % kLanes));
        if (r != LZ4B200_OK) return r;
        scan_sizes_kernel<<<1, 1024, 0, ln.stream>>>(ctx->d_out_len.p + c.b0, ctx->d_seg_off.p + c.b0 + ci, n);
        CTX_CUDA(ctx, cudaGetLastError());
        CTX_CUDA(ctx, cudaMemcpyAsync(pl.h_seg + c.b0 + ci, ctx->d_seg_off.p + c.b0 + ci, (n + 1) * 8,
                                      cudaMemcpyDeviceToHost, ln.stream));
        CTX_CUDA(ctx, cudaEventRecord(ln.sizes_ready, ln.stream));
        return LZ4B200_OK;
    };

    for (uint32_t ci = 0; ci < nch && ci < (uint32_t)kLanes; ci++) {
        st = phase1(ci);
        if (st != LZ4B200_OK) return st;
    }
    uint64_t out_base = 0;
    lz4b200_status result = LZ4B200_OK;
    for (uint32_t ci = 0; ci < nch; ci++) {
        const Chunk &c = chunks[ci];
        Lane &ln = pl.lane[ci % kLanes];
        const uint32_t n = c.b1 - c.b0;
        CTX_CUDA(ctx, cudaEventSynchronize(ln.sizes_ready));
        const uint64_t *seg = pl.h_seg + c.b0 + ci;
        const uint64_t total = seg[n];
        for (uint32_t k = 0; k < n; k++) {
            out_off[c.b0 + k] = out_base + seg[k];
            out_len[c.b0 + k] = (uint32_t)(seg[k + 1] - seg[k]);
        }
        if (out_base + total > out_cap_total) { result = LZ4B200_COMPRESS_OUTPUT_TOO_SMALL; break; }
        if (total) {
            CTX_CUDA(ctx, ln.out.reserve(total + 16));
            GatherArgs g{ln.slots.p, nullptr, ctx->d_out_off.p + c.b0, nullptr, ctx->d_out_len.p + c.b0, nullptr, nullptr,
                         nullptr, ln.out.p, ctx->d_seg_off.p + c.b0 + ci, n};
            gather_segments_kernel<<<std::min<uint32_t>(n, (uint32_t)ctx->sm_count * 8), 256, 0, ln.stream>>>(g);
            CTX_CUDA(ctx, cudaGetLastError());
            CTX_CUDA(ctx, cudaMemcpyAsync(out + out_base, ln.out.p, total, cudaMemcpyDeviceToHost, ln.stream));
        }
        out_base += total;
        if (ci + kLanes < nch) {
            st = phase1(ci + kLanes);
            if (st != LZ4B200_OK) return st;
        }
    }
    for (int i = 0; i < kLanes; i++) CTX_CUDA(ctx, cudaStreamSynchronize(pl.lane[i].stream));
    if (result != LZ4B200_OK) return result;
    CTX_CUDA(ctx, cudaMemcpyAsync(pl.h_status, ctx->d_status.p, nb * 4, cudaMemcpyDeviceToHost, s0));
    CTX_CUDA(ctx, cudaStreamSynchronize(s0));
    memcpy(status, pl.h_status, nb * 4);
    return LZ4B200_OK;
}

static lz4b200_status decompress_batch_host_impl(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                                 const uint32_t *in_len, const uint8_t *dict, size_t dict_len,
                                                 uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
                                                 uint32_t *out_len, int32_t *status, uint64_t *err_expected,
                                                 size_t nblocks)
{
    if (!ctx || nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (nblocks == 0) return LZ4B200_OK;
    if (!in || !in_off || !in_len || !out || !out_off || !out_cap || !out_len || !status)
        return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    Pipeline &pl = ctx_pipeline(ctx);
    const int kLanes = lanes_in_use();
    lz4b200_status st = pipeline_init(ctx, pl);
    if (st != LZ4B200_OK) return st;
    const uint32_t nb = (uint32_t)nblocks;

    static const uint64_t kChunkBytes = env_mib("LZ4B200_DEC_CHUNK_MB", kChunkBytesDefault);
    std::vector<Chunk> chunks;
    std::vector<uint8_t> contiguous;
    std::vector<uint64_t> h_in_off(nb), h_out_off(nb);
    for (uint32_t b = 0; b < nb;) {
        Chunk c{b, b, ~0ull, 0, ~0ull, 0};
        uint64_t bytes = 0;
        bool contig = true;
        const uint64_t limit = std::min<uint64_t>(kChunkBytes, (32ull << 20) << std::min<size_t>(chunks.size(), 8));
        while (c.b1 < nb && (c.b1 == c.b0 || bytes + out_cap[c.b1] <= limit)) {
            const uint32_t k = c.b1++;
            c.in_lo = std::min<uint64_t>(c.in_lo, in_off[k]); c.in_hi = std::max<uint64_t>(c.in_hi, in_off[k] + in_len[k]);
            c.a = std::min<uint64_t>(c.a, out_off[k]); c.b = std::max<uint64_t>(c.b, out_off[k] + out_cap[k]);
            if (k > c.b0 && out_off[k] != out_off[k - 1] + out_cap[k - 1]) contig = false;
            bytes += out_cap[k];
        }
        for (uint32_t k = c.b0; k < c.b1; k++) { h_in_off[k] = in_off[k] - c.in_lo; h_out_off[k] = out_off[k] - c.a; }
        chunks.push_back(c);
        contiguous.push_back(contig ? 1 : 0);
        b = c.b1;
    }
    const uint32_t nch = (uint32_t)chunks.size();
    CTX_CUDA(ctx, ctx->d_in_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_in_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_status.reserve(nb));
    CTX_CUDA(ctx, ctx->d_expected.reserve(nb));
    CTX_CUDA(ctx, pinned_reserve(pl.h_seg, pl.h_seg_cap, (size_t)nb));
    CTX_CUDA(ctx, pinned_reserve(pl.h_status, pl.h_status_cap, (size_t)nb * 2));
    cudaStream_t s0 = pl.lane[0].stream;
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_off.p, h_in_off.data(), nb * 8, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_len.p, in_len, nb * 4, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_off.p, h_out_off.data(), nb * 8, cudaMemcpyHostToDevice, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_cap.p, out_cap, nb * 4, cudaMemcpyHostToDevice, s0));
    normalize_dict(dict, dict_len, false);
    if (dict_len) {
        CTX_CUDA(ctx, ctx->d_dict.reserve(dict_len + 16));
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_dict.p, dict, dict_len, cudaMemcpyHostToDevice, s0));
    }
    CTX_CUDA(ctx, cudaEventRecord(pl.desc_ready, s0));
    CTX_CUDA(ctx, cudaStreamSynchronize(s0));

    for (uint32_t ci = 0; ci < nch; ci++) {
        const Chunk &c = chunks[ci];
        Lane &ln = pl.lane[ci % kLanes];
        const uint32_t n = c.b1 - c.b0;
        CTX_CUDA(ctx, ln.in.reserve(c.in_hi - c.in_lo + 16));
        CTX_CUDA(ctx, ln.out.reserve(c.b - c.a + 16));
        CTX_CUDA(ctx, cudaStreamWaitEvent(ln.stream, pl.desc_ready, 0));
        CTX_CUDA(ctx, cudaMemcpyAsync(ln.in.p, in + c.in_lo, c.in_hi - c.in_lo, cudaMemcpyHostToDevice, ln.stream));
        // The whole capacity region of every slot travels back (the decoded sizes are only known after the kernel), so
        // what lies past a block's decoded length must not be whatever an earlier call left in this staging buffer.
        CTX_CUDA(ctx, cudaMemsetAsync(ln.out.p, 0, c.b - c.a, ln.stream));
        BatchArgs a{ln.in.p, ctx->d_in_off.p + c.b0, ctx->d_in_len.p + c.b0, nullptr, ln.out.p, ctx->d_out_off.p + c.b0,
                    ctx->d_out_cap.p + c.b0, ctx->d_out_len.p + c.b0, ctx->d_status.p + c.b0, ctx->d_expected.p + c.b0, n,
                    nullptr};
        if (dict_len) { a.dict = ctx->d_dict.p; a.dict_len = (uint32_t)dict_len; }
        st = launch_decompress(ctx, a, ln.stream, pl.d_tickets + 8 * (ci % kLanes));
        if (st != LZ4B200_OK) return st;
        if (contiguous[ci]) {
            CTX_CUDA(ctx, cudaMemcpyAsync(out + c.a, ln.out.p, c.b - c.a, cudaMemcpyDeviceToHost, ln.stream));
        } else {
            for (uint32_t k = c.b0; k < c.b1; k++)
                if (out_cap[k])
                    CTX_CUDA(ctx, cudaMemcpyAsync(out + out_off[k], ln.out.p + h_out_off[k], out_cap[k],
                                                  cudaMemcpyDeviceToHost, ln.stream));
        }
    }
    for (int i = 0; i < kLanes; i++) CTX_CUDA(ctx, cudaStreamSynchronize(pl.lane[i].stream));
    uint32_t *h_len = reinterpret_cast<uint32_t *>(pl.h_status + nb);
    CTX_CUDA(ctx, cudaMemcpyAsync(pl.h_status, ctx->d_status.p, nb * 4, cudaMemcpyDeviceToHost, s0));
    CTX_CUDA(ctx, cudaMemcpyAsync(h_len, ctx->d_out_len.p, nb * 4, cudaMemcpyDeviceToHost, s0));
    if (err_expected)
        CTX_CUDA(ctx, cudaMemcpyAsync(pl.h_seg, ctx->d_expected.p, nb * 8, cudaMemcpyDeviceToHost, s0));
    CTX_CUDA(ctx, cudaStreamSynchronize(s0));
    memcpy(status, pl.h_status, nb * 4);
    memcpy(out_len, h_len, nb * 4);
    if (err_expected) memcpy(err_expected, pl.h_seg, nb * 8);
    return LZ4B200_OK;
}

extern "C" {

lz4b200_status lz4b200_compress_batch_host(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                           const uint32_t *in_len, const uint8_t *flags, uint8_t *out,
                                           size_t out_cap_total, uint64_t *out_off, uint32_t *out_len,
                                           int32_t *status, size_t nblocks)
{
    return compress_batch_host_impl(ctx, in, in_off, in_len, flags, nullptr, 0, out, out_cap_total, out_off, out_len,
                                    status, nblocks);
}

lz4b200_status lz4b200_decompress_batch_host(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                             const uint32_t *in_len, uint8_t *out, const uint64_t *out_off,
                                             const uint32_t *out_cap, uint32_t *out_len, int32_t *status,
                                             uint64_t *err_expected, size_t nblocks)
{
    return decompress_batch_host_impl(ctx, in, in_off, in_len, nullptr, 0, out, out_off, out_cap, out_len, status,
                                      err_expected, nblocks);
}

lz4b200_status lz4b200_compress_batch_host_with_dict(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                                     const uint32_t *in_len, const uint8_t *dict, size_t dict_len,
                                                     uint8_t *out, size_t out_cap_total, uint64_t *out_off,
                                                     uint32_t *out_len, int32_t *status, size_t nblocks)
{
    return compress_batch_host_impl(ctx, in, in_off, in_len, nullptr, dict, dict_len, out, out_cap_total, out_off,
                                    out_len, status, nblocks);
}

lz4b200_status lz4b200_decompress_batch_host_with_dict(lz4b200_ctx *ctx, const uint8_t *in, const uint64_t *in_off,
                                                       const uint32_t *in_len, const uint8_t *dict, size_t dict_len,
                                                       uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
                                                       uint32_t *out_len, int32_t *status, uint64_t *err_expected,
                                                       size_t nblocks)
{
    return decompress_batch_host_impl(ctx, in, in_off, in_len, dict, dict_len, out, out_off, out_cap, out_len, status,
                                      err_expected, nblocks);
}

// ---- single-block host entry points -----------------------------------------------------------

lz4b200_status lz4b200_compress_into(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                     size_t *written)
{
    if (!ctx || !written || (!in && n) || n > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (cap < lz4b200_max_output_size(n)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;     // compress.rs:338-340
    uint64_t in_off = 0, out_off = 0;
    uint32_t in_len = (uint32_t)n, out_len = 0;
    int32_t status = 0;
    static const uint8_t zero = 0;
    lz4b200_status st = lz4b200_compress_batch_host(ctx, n ? in : &zero, &in_off, &in_len, nullptr, out, cap, &out_off,
                                                    &out_len, &status, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) return (lz4b200_status)status;
    *written = out_len;
    return LZ4B200_OK;
}

lz4b200_status lz4b200_compress_prepend_size(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                             size_t *written)
{
    if (!written) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (cap < 4) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    wr32(out, (uint32_t)n);                                                              // compress.rs:633/649
    size_t w = 0;
    lz4b200_status st = lz4b200_compress_into(ctx, in, n, out + 4, cap - 4, &w);
    if (st == LZ4B200_OK) *written = w + 4;
    return st;
}

lz4b200_status lz4b200_decompress_into(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                       size_t *written, size_t *err_expected, size_t *err_actual)
{
    if (!ctx || !written || n > 0xffffffffull || cap > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (err_expected) *err_expected = 0;
    if (err_actual) *err_actual = 0;
    if (n == 0) return LZ4B200_DEC_EXPECTED_ANOTHER_BYTE;                                // decompress.rs:207-209
    uint64_t in_off = 0, out_off = 0, expected = 0;
    uint32_t in_len = (uint32_t)n, out_cap = (uint32_t)cap, out_len = 0;
    int32_t status = 0;
    uint8_t dummy = 0;
    lz4b200_status st = lz4b200_decompress_batch_host(ctx, in, &in_off, &in_len, cap ? out : &dummy, &out_off, &out_cap,
                                                      &out_len, &status, &expected, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) {
        if (status == LZ4B200_DEC_OUTPUT_TOO_SMALL) {
            if (err_expected) *err_expected = (size_t)expected;
            if (err_actual) *err_actual = cap;
        }
        return (lz4b200_status)status;
    }
    *written = out_len;
    return LZ4B200_OK;
}

// ---- external dictionary (compress.rs:610-616, 685-693; decompress.rs:462-468, 478-528) ------------------

lz4b200_status lz4b200_compress_into_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n, const uint8_t *dict,
                                               size_t dict_len, uint8_t *out, size_t cap, size_t *written)
{
    if (!ctx || !written || (!in && n) || n > 0xffffffffull || (!dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (cap < lz4b200_max_output_size(n)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;     // compress.rs:338-340
    uint64_t in_off = 0, out_off = 0;
    uint32_t in_len = (uint32_t)n, out_len = 0;
    int32_t status = 0;
    static const uint8_t zero = 0;
    lz4b200_status st = compress_batch_host_impl(ctx, n ? in : &zero, &in_off, &in_len, nullptr, dict, dict_len, out, cap,
                                                 &out_off, &out_len, &status, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) return (lz4b200_status)status;
    *written = out_len;
    return LZ4B200_OK;
}

// block::compress_into_with_table (compress.rs:744-766).  The reusable CompressTable only decides which table
// layout / hash the parse uses: Small = u16 entries + 4-byte hash (inputs < 65 535 bytes), Large = u32 entries +
// 5-byte hash for any size; a Small table handed an input >= 65 535 bytes is upgraded to Large and stays Large.
// *table_kind carries that state (LZ4B200_TABLE_SMALL / LZ4B200_TABLE_LARGE); the table's memory lives on the GPU.
lz4b200_status lz4b200_compress_into_with_table(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                                size_t *written, int *table_kind)
{
    if (!ctx || !written || !table_kind || (!in && n) || n > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    if (*table_kind != LZ4B200_TABLE_SMALL && *table_kind != LZ4B200_TABLE_LARGE) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (n >= 65535 && *table_kind == LZ4B200_TABLE_SMALL) *table_kind = LZ4B200_TABLE_LARGE;      // compress.rs:750-752
    if (cap < lz4b200_max_output_size(n)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;                // compress.rs:338-340
    uint64_t in_off = 0, out_off = 0;
    uint32_t in_len = (uint32_t)n, out_len = 0;
    int32_t status = 0;
    const uint8_t flag = *table_kind == LZ4B200_TABLE_LARGE ? (uint8_t)LZ4B200_BLOCK_HASH5_ALWAYS : (uint8_t)0;
    static const uint8_t zero = 0;
    lz4b200_status st = compress_batch_host_impl(ctx, n ? in : &zero, &in_off, &in_len, &flag, nullptr, 0, out, cap,
                                                 &out_off, &out_len, &status, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) return (lz4b200_status)status;
    *written = out_len;
    return LZ4B200_OK;
}

lz4b200_status lz4b200_compress_prepend_size_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                       const uint8_t *dict, size_t dict_len, uint8_t *out, size_t cap,
                                                       size_t *written)
{
    if (!written) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (cap < 4) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    wr32(out, (uint32_t)n);
    size_t w = 0;
    lz4b200_status st = lz4b200_compress_into_with_dict(ctx, in, n, dict, dict_len, out + 4, cap - 4, &w);
    if (st == LZ4B200_OK) *written = w + 4;
    return st;
}

lz4b200_status lz4b200_decompress_into_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n, const uint8_t *dict,
                                                 size_t dict_len, uint8_t *out, size_t cap, size_t *written,
                                                 size_t *err_expected, size_t *err_actual)
{
    if (!ctx || !written || n > 0xffffffffull || cap > 0xffffffffull || (!dict && dict_len)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (err_expected) *err_expected = 0;
    if (err_actual) *err_actual = 0;
    if (n == 0) return LZ4B200_DEC_EXPECTED_ANOTHER_BYTE;                                // decompress.rs:207-209
    uint64_t in_off = 0, out_off = 0, expected = 0;
    uint32_t in_len = (uint32_t)n, out_cap = (uint32_t)cap, out_len = 0;
    int32_t status = 0;
    uint8_t dummy = 0;
    lz4b200_status st = decompress_batch_host_impl(ctx, in, &in_off, &in_len, dict, dict_len, cap ? out : &dummy, &out_off,
                                                   &out_cap, &out_len, &status, &expected, 1);
    if (st != LZ4B200_OK) return st;
    if (status != LZ4B200_OK) {
        if (status == LZ4B200_DEC_OUTPUT_TOO_SMALL) {
            if (err_expected) *err_expected = (size_t)expected;
            if (err_actual) *err_actual = cap;
        }
        return (lz4b200_status)status;
    }
    *written = out_len;
    return LZ4B200_OK;
}

lz4b200_status lz4b200_decompress_size_prepended_with_dict(lz4b200_ctx *ctx, const uint8_t *in, size_t n,
                                                           const uint8_t *dict, size_t dict_len, uint8_t *out,
                                                           size_t cap, size_t *written, size_t *err_expected,
                                                           size_t *err_actual)
{
    size_t want = 0;
    if (written) *written = 0;
    lz4b200_status st = lz4b200_uncompressed_size(in, n, &want);
    if (st != LZ4B200_OK) return st;
    if (cap < want) return LZ4B200_INVALID_ARGUMENT;
    return lz4b200_decompress_into_with_dict(ctx, in + 4, n - 4, dict, dict_len, out, want, written, err_expected,
                                             err_actual);
}

lz4b200_status lz4b200_uncompressed_size(const uint8_t *in, size_t n, size_t *size)
{
    if (!size) return LZ4B200_INVALID_ARGUMENT;
    if (n < 4) return LZ4B200_DEC_EXPECTED_ANOTHER_BYTE;                                 // block/mod.rs:151-157
    *size = rd32(in);
    return LZ4B200_OK;
}

lz4b200_status lz4b200_decompress_size_prepended(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out,
                                                 size_t cap, size_t *written, size_t *err_expected,
                                                 size_t *err_actual)
{
    size_t want = 0;
    if (written) *written = 0;
    lz4b200_status st = lz4b200_uncompressed_size(in, n, &want);
    if (st != LZ4B200_OK) return st;
    if (cap < want) return LZ4B200_INVALID_ARGUMENT;
    return lz4b200_decompress_into(ctx, in + 4, n - 4, out, want, written, err_expected, err_actual);
}

// ---- frame format ---------------------------------------------------------------------------------

size_t lz4b200_frame_write_header(const lz4b200_frame_info *info, uint8_t *out, size_t cap)
{
    // FrameInfo::write — frame/header.rs:232-275
    uint8_t buf[19];
    size_t o = 0;
    wr32(buf, 0x184D2204u); o = 4;
    uint8_t flg = 0x40;
    if (info->block_checksums) flg |= 0x10;
    if (info->content_checksum) flg |= 0x04;
    if (!info->linked) flg |= 0x20;
    if (info->has_content_size) flg |= 0x08;
    buf[o++] = flg;
    buf[o++] = (uint8_t)(info->block_size_id << 4);
    if (info->has_content_size) { memcpy(buf + o, &info->content_size, 8); o += 8; }
    buf[o] = (uint8_t)(lz4b200_xxh32(buf + 4, o - 4, 0) >> 8);
    o++;
    if (cap < o) return 0;
    memcpy(out, buf, o);
    return o;
}

size_t lz4b200_frame_blocks_bound(size_t in_len, size_t block_size)
{
    size_t nb = block_size ? (in_len + block_size - 1) / block_size : 0;
    return in_len + nb * 4;
}

size_t lz4b200_frame_bound(size_t n, const lz4b200_frame_info *info)
{
    int id = info && info->block_size_id ? info->block_size_id : 4;
    size_t bs = block_size_bytes(id);
    if (!bs) bs = 64u << 10;
    size_t nb = (n + bs - 1) / bs;
    return 19 + n + nb * 8 + 8;
}

// Rank-local half of a (possibly sharded) frame, step 1: compress the blocks of [first_block, ...) into the context's
// slots, decide compressed-vs-stored per block (frame/compress.rs:301-306) and scan the segment sizes.  *d_total
// receives the packed size.  Everything stays on the device and on `stream`.
lz4b200_status lz4b200_frame_range_compress(lz4b200_ctx *ctx, const uint8_t *d_in, size_t in_len, size_t block_size,
                                            uint64_t first_block, uint64_t *d_total, uint32_t *d_block_sizes, void *stream)
{
    if (!ctx || !block_size || block_size > (8u << 20)) return LZ4B200_INVALID_ARGUMENT;
    const size_t nblocks = (in_len + block_size - 1) / block_size;
    if (nblocks > 0xffffffffull) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nb = (uint32_t)nblocks;
    ctx->range_nb = nb; ctx->range_in = d_in;
    if (nb == 0) {
        if (d_total) CTX_CUDA(ctx, cudaMemsetAsync(d_total, 0, 8, s));
        return LZ4B200_OK;
    }
    const size_t slot = (lz4b200_max_output_size(block_size) + 15) & ~size_t(15);
    CTX_CUDA(ctx, ctx->d_slots.reserve(slot * nb + 16));
    CTX_CUDA(ctx, ctx->d_in_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_in_len.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_off.reserve(nb)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(nb));
    CTX_CUDA(ctx, ctx->d_out_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_status.reserve(nb));
    CTX_CUDA(ctx, ctx->d_flags.reserve(nb)); CTX_CUDA(ctx, ctx->d_pick.reserve(nb));
    CTX_CUDA(ctx, ctx->d_info.reserve(nb)); CTX_CUDA(ctx, ctx->d_seg_size.reserve(nb));
    CTX_CUDA(ctx, ctx->d_payload_len.reserve(nb)); CTX_CUDA(ctx, ctx->d_seg_off.reserve(nb + 1));

    make_uniform_desc_kernel<<<(nb + 255) / 256, 256, 0, s>>>(in_len, (uint32_t)block_size, slot, first_block,
                                                             fresh_period(block_size), nb, ctx->d_in_off.p,
                                                             ctx->d_in_len.p, ctx->d_out_off.p, ctx->d_out_cap.p,
                                                             ctx->d_flags.p);
    CTX_CUDA(ctx, cudaGetLastError());
    BatchArgs a{d_in, ctx->d_in_off.p, ctx->d_in_len.p, ctx->d_flags.p, ctx->d_slots.p, ctx->d_out_off.p,
                ctx->d_out_cap.p, ctx->d_out_len.p, ctx->d_status.p, nullptr, nb, nullptr};
    lz4b200_status st = launch_compress(ctx, a, (uint32_t)std::min<size_t>(block_size, in_len), s);
    if (st != LZ4B200_OK) return st;
    frame_block_info_kernel<<<(nb + 255) / 256, 256, 0, s>>>(ctx->d_out_len.p, ctx->d_in_len.p, nb, ctx->d_info.p,
                                                            ctx->d_pick.p, ctx->d_seg_size.p, ctx->d_payload_len.p);
    CTX_CUDA(ctx, cudaGetLastError());
    scan_sizes_kernel<<<1, 1024, 0, s>>>(ctx->d_seg_size.p, ctx->d_seg_off.p, nb);
    CTX_CUDA(ctx, cudaGetLastError());
    if (d_total) CTX_CUDA(ctx, cudaMemcpyAsync(d_total, ctx->d_seg_off.p + nb, 8, cudaMemcpyDeviceToDevice, s));
    if (d_block_sizes)
        CTX_CUDA(ctx, cudaMemcpyAsync(d_block_sizes, ctx->d_seg_size.p, nb * 4, cudaMemcpyDeviceToDevice, s));
    return LZ4B200_OK;
}

// Step 2: pack the range's [BlockInfo | payload] segments back to back at d_dst + *d_dst_offset.  d_dst may be PEER
// memory (another GPU's frame buffer mapped over NVLink, lz4b200_peer_open): the pack kernel's stores are then the
// transfer — the per-rank chunk is never staged in local memory or handed to a separate collective.
lz4b200_status lz4b200_frame_range_pack(lz4b200_ctx *ctx, uint8_t *d_dst, const uint64_t *d_dst_offset, void *stream)
{
    if (!ctx || !d_dst) return LZ4B200_INVALID_ARGUMENT;
    const uint32_t nb = ctx->range_nb;
    if (nb == 0) return LZ4B200_OK;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = (cudaStream_t)stream;
    GatherArgs g{ctx->d_slots.p, ctx->range_in, ctx->d_out_off.p, ctx->d_in_off.p, ctx->d_payload_len.p, ctx->d_payload_len.p,
                 ctx->d_pick.p, ctx->d_info.p, d_dst, ctx->d_seg_off.p, nb, d_dst_offset};
    gather_segments_kernel<<<std::min<uint32_t>(std::max<uint32_t>(nb, (uint32_t)ctx->sm_count * 2), (uint32_t)ctx->sm_count * 8),
                             256, 0, s>>>(g);
    CTX_CUDA(ctx, cudaGetLastError());
    return LZ4B200_OK;
}

lz4b200_status lz4b200_frame_compress_blocks_device(lz4b200_ctx *ctx, const uint8_t *d_in, size_t in_len,
                                                    size_t block_size, uint64_t first_block, uint8_t *d_out,
                                                    size_t out_cap, uint64_t *d_total, uint32_t *d_block_sizes,
                                                    void *stream)
{
    if (!ctx || !block_size || block_size > (8u << 20)) return LZ4B200_INVALID_ARGUMENT;
    if (out_cap < lz4b200_frame_blocks_bound(in_len, block_size)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    lz4b200_status st = lz4b200_frame_range_compress(ctx, d_in, in_len, block_size, first_block, d_total, d_block_sizes, stream);
    if (st != LZ4B200_OK || in_len == 0) return st;
    return lz4b200_frame_range_pack(ctx, d_out, nullptr, stream);
}

// ---- peer-mapped buffers (CUDA IPC): rank 0 allocates the frame buffer, the other ranks of the node map it ----------
lz4b200_status lz4b200_peer_alloc(lz4b200_ctx *ctx, size_t bytes, void **d_ptr, uint8_t *handle64)
{
    if (!ctx || !d_ptr || !handle64 || !bytes) return LZ4B200_INVALID_ARGUMENT;
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
    DeviceGuard guard(ctx->device);
    void *p = nullptr;
    CTX_CUDA(ctx, cudaMalloc(&p, bytes));
    cudaIpcMemHandle_t h;
    if (!ctx->check(cudaIpcGetMemHandle(&h, p), "cudaIpcGetMemHandle")) { cudaFree(p); return LZ4B200_CUDA_ERROR; }
    memcpy(handle64, &h, 64);
    *d_ptr = p;
    return LZ4B200_OK;
}

lz4b200_status lz4b200_peer_open(lz4b200_ctx *ctx, const uint8_t *handle64, void **d_ptr)
{
    if (!ctx || !d_ptr || !handle64) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    cudaIpcMemHandle_t h;
    memcpy(&h, handle64, 64);
    CTX_CUDA(ctx, cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return LZ4B200_OK;
}

lz4b200_status lz4b200_peer_close(lz4b200_ctx *ctx, void *d_ptr)
{
    if (!ctx || !d_ptr) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    CTX_CUDA(ctx, cudaIpcCloseMemHandle(d_ptr));
    return LZ4B200_OK;
}

lz4b200_status lz4b200_peer_free(lz4b200_ctx *ctx, void *d_ptr)
{
    if (!ctx || !d_ptr) return LZ4B200_INVALID_ARGUMENT;
    DeviceGuard guard(ctx->device);
    CTX_CUDA(ctx, cudaFree(d_ptr));
    return LZ4B200_OK;
}

lz4b200_status lz4b200_frame_compress(lz4b200_ctx *ctx, const uint8_t *in, size_t n, const lz4b200_frame_info *info_in,
                                      size_t first_write_len, uint8_t *out, size_t cap, size_t *written)
{
    if (!ctx || !info_in || !out || !written || (!in && n)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    lz4b200_frame_info info = *info_in;
    if (info.linked) return LZ4B200_FRAME_LINKED_UNSUPPORTED;
    if (info.block_size_id == 0) info.block_size_id = auto_block_size_id(first_write_len);   // compress.rs:236-238
    if (info.block_size_id < 4 || info.block_size_id > 7) return LZ4B200_INVALID_ARGUMENT;
    if (info.has_content_size && info.content_size != n) return LZ4B200_FRAME_CONTENT_LENGTH; // compress.rs:212-219
    const size_t bs = block_size_bytes(info.block_size_id);
    if (cap < lz4b200_frame_bound(n, &info)) return LZ4B200_COMPRESS_OUTPUT_TOO_SMALL;
    DeviceGuard guard(ctx->device);
    cudaStream_t s = ctx->stream;

    size_t o = lz4b200_frame_write_header(&info, out, cap);
    const size_t nblocks = (n + bs - 1) / bs;
    if (nblocks) {
        const size_t bound = lz4b200_frame_blocks_bound(n, bs);
        CTX_CUDA(ctx, ctx->d_in.reserve(n + 16));
        CTX_CUDA(ctx, ctx->d_out.reserve(bound + 16));
        CTX_CUDA(ctx, ctx->d_off_b.reserve(1));
        CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in.p, in, n, cudaMemcpyHostToDevice, s));
        lz4b200_status st = lz4b200_frame_compress_blocks_device(ctx, ctx->d_in.p, n, bs, 0, ctx->d_out.p, bound,
                                                                 ctx->d_off_b.p, nullptr, s);
        if (st != LZ4B200_OK) return st;
        uint64_t total = 0;
        CTX_CUDA(ctx, cudaMemcpyAsync(&total, ctx->d_off_b.p, 8, cudaMemcpyDeviceToHost, s));
        CTX_CUDA(ctx, cudaStreamSynchronize(s));
        if (!info.block_checksums) {
            CTX_CUDA(ctx, cudaMemcpyAsync(out + o, ctx->d_out.p, total, cudaMemcpyDeviceToHost, s));
            CTX_CUDA(ctx, cudaStreamSynchronize(s));
            o += total;
        } else {
            // block checksum = XXH32 of the payload as written (frame/compress.rs:313-316): host-side walk
            std::vector<uint8_t> tmp(total);
            CTX_CUDA(ctx, cudaMemcpyAsync(tmp.data(), ctx->d_out.p, total, cudaMemcpyDeviceToHost, s));
            CTX_CUDA(ctx, cudaStreamSynchronize(s));
            size_t p = 0;
            while (p < total) {
                uint32_t word = rd32(tmp.data() + p);
                size_t len = word & 0x7fffffffu;
                memcpy(out + o, tmp.data() + p, 4 + len);
                wr32(out + o + 4 + len, lz4b200_xxh32(tmp.data() + p + 4, len, 0));
                o += 8 + len; p += 4 + len;
            }
        }
    }
    wr32(out + o, 0); o += 4;                                                            // EndMark: compress.rs:221-223
    if (info.content_checksum) { wr32(out + o, lz4b200_xxh32(in, n, 0)); o += 4; }       // compress.rs:224-227
    *written = o;
    return LZ4B200_OK;
}

namespace {

struct FrameBlockRef {
    uint64_t payload_off;     // into the input buffer
    uint32_t payload_len;
    uint32_t max_out;         // block size of the owning frame
    bool stored;
    uint32_t frame_idx;
};
struct FrameRef {
    uint32_t first_block, nblocks;
    bool has_size, has_checksum, closed;
    bool linked = false;      // BlockMode::Linked: blocks may reference the frame's earlier output
    uint64_t content_size;
    uint32_t content_checksum;
};

}  // namespace

// Upper bound of what one block can decode to: its frame's block size, and never more than 255 output bytes per
// input byte (a length-extension byte of 0xFF stands for 255 bytes; nothing in the format is denser).
static inline uint64_t block_decoded_cap(uint64_t payload_len, uint64_t bs)
{
    return std::min<uint64_t>(bs, payload_len * 255ull + 16ull);
}

lz4b200_status lz4b200_frame_decoded_bound(const uint8_t *in, size_t n, size_t *bound)
{
    if (!bound || (!in && n)) return LZ4B200_INVALID_ARGUMENT;
    size_t ip = 0, total = 0;
    while (ip + 4 <= n) {
        uint32_t magic = rd32(in + ip);
        size_t bs; unsigned flg = 0x20;
        if (magic == 0x184C2102u) { ip += 4; bs = 8u << 20; }
        else {
            if (n - ip < 7 || magic != 0x184D2204u) break;
            flg = in[ip + 4];
            int id = (in[ip + 5] >> 4) & 7;
            bs = block_size_bytes(id);
            if (!bs) break;
            size_t need = 7 + ((flg & 8) ? 8 : 0) + ((flg & 1) ? 4 : 0);
            if (n - ip < need) break;
            ip += need;
        }
        // The header's content_size is NOT used: it is untrusted, and a frame whose real size differs must still be
        // delivered in full before ContentLengthError is reported (frame/decompress.rs:312-321).
        for (;;) {
            if (n - ip < 4) { ip = n; break; }
            uint32_t word = rd32(in + ip); ip += 4;
            if (word == 0) { if (flg & 4) ip += 4; break; }
            size_t len = word & 0x7fffffffu;
            total += (word & 0x80000000u) ? len : (size_t)block_decoded_cap(len, bs);
            ip += len + ((flg & 0x10) ? 4 : 0);
            if (ip > n) { ip = n; break; }
        }
    }
    *bound = total;
    return LZ4B200_OK;
}

void lz4b200_ctx_set_frame_budget(lz4b200_ctx *ctx, size_t bytes)
{
    if (ctx) ctx->frame_budget = std::max<size_t>(bytes, 1u << 20);
}

// One frame.  Host walk of its header and BlockInfo chain (frame/decompress.rs:109-342), then the blocks are decoded
// in groups whose device slots fit the context's frame budget (slots are reused from group to group), so a frame of
// many short blocks costs O(budget) device memory, not #blocks x block size.
lz4b200_status lz4b200_frame_decompress_next(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                             size_t *consumed, size_t *written, int *block_status,
                                             uint64_t *err_expected, uint64_t *err_actual)
{
    if (!ctx || !written || !consumed || (!in && n) || (!out && cap)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0; *consumed = 0;
    if (block_status) *block_status = 0;
    if (err_expected) *err_expected = 0;
    if (err_actual) *err_actual = 0;
    if (n == 0) return LZ4B200_OK;                          // read_frame_info: 0 bytes where a frame would start = end of data

    // ---- header -----------------------------------------------------------------------------------
    std::vector<FrameBlockRef> blocks;
    lz4b200_status walk_err = LZ4B200_OK;
    size_t ip = 0;
    size_t bs; unsigned flg = 0x20;
    FrameRef fr{0, 0, false, false, false, 0, 0};
    if (n < 4) { *consumed = n; return LZ4B200_FRAME_IO_EOF; }
    const uint32_t magic = rd32(in);
    if (magic == 0x184C2102u) {                             // legacy frame: header.rs:285-291
        ip = 4; bs = 8u << 20;
    } else {
        if (n == 4) { *consumed = 4; return LZ4B200_OK; }   // decompress.rs:124-128: nothing after the magic = end of data
        if (n < 7) { *consumed = n; return LZ4B200_FRAME_IO_EOF; }
        if (magic >= 0x184D2A50u && magic <= 0x184D2A5Fu) return LZ4B200_FRAME_SKIPPABLE;
        if (magic != 0x184D2204u) return LZ4B200_FRAME_WRONG_MAGIC;
        flg = in[4];
        const uint8_t bd = in[5];
        const size_t need = 7 + ((flg & 0x08) ? 8 : 0) + ((flg & 0x01) ? 4 : 0);
        if (n < need) { *consumed = n; return LZ4B200_FRAME_IO_EOF; }
        if ((flg & 0xC0) != 0x40) return LZ4B200_FRAME_UNSUPPORTED_VERSION;
        if ((flg & 0x02) || (bd & 0x8F)) return LZ4B200_FRAME_RESERVED_BITS;
        const int id = (bd >> 4) & 7;
        if (id < 4) return LZ4B200_FRAME_UNSUPPORTED_BLOCKSIZE;
        bs = block_size_bytes(id);
        size_t o = 6;
        if (flg & 0x08) { memcpy(&fr.content_size, in + o, 8); fr.has_size = true; o += 8; }
        if (flg & 0x01) o += 4;
        if ((uint8_t)(lz4b200_xxh32(in + 4, o - 4, 0) >> 8) != in[o]) return LZ4B200_FRAME_HEADER_CHECKSUM;
        if (flg & 0x01) return LZ4B200_FRAME_DICTIONARY;
        fr.linked = !(flg & 0x20);
        ip = o + 1;
    }
    // ---- BlockInfo chain --------------------------------------------------------------------------
    for (;;) {
        if (n - ip < 4) { ip = n; break; }                  // EOF where a BlockInfo is due: decompress.rs:236-243
        const uint32_t word = rd32(in + ip); ip += 4;
        if (word == 0) {                                     // EndMark
            fr.closed = true;
            if (flg & 0x04) {
                if (n - ip < 4) { walk_err = LZ4B200_FRAME_IO_EOF; ip = n; break; }
                fr.has_checksum = true; fr.content_checksum = rd32(in + ip); ip += 4;
            }
            break;
        }
        const size_t len = word & 0x7fffffffu;
        if (len > bs) { walk_err = LZ4B200_FRAME_BLOCK_TOO_BIG; break; }
        if (n - ip < len) { walk_err = LZ4B200_FRAME_IO_EOF; ip = n; break; }
        const size_t payload = ip; ip += len;
        if (flg & 0x10) {
            if (n - ip < 4) { walk_err = LZ4B200_FRAME_IO_EOF; ip = n; break; }
            if (rd32(in + ip) != lz4b200_xxh32(in + payload, len, 0)) { walk_err = LZ4B200_FRAME_BLOCK_CHECKSUM; break; }
            ip += 4;
        }
        blocks.push_back({payload, (uint32_t)len, (uint32_t)bs, (word & 0x80000000u) != 0, 0});
        fr.nblocks++;
    }
    *consumed = ip;

    // ---- decode every block seen before the walk stopped, group by group ---------------------------
    const uint32_t nb = (uint32_t)blocks.size();
    uint64_t total = 0;
    Xxh32 content(0);
    if (nb) {
        DeviceGuard guard(ctx->device);
        cudaStream_t s = ctx->stream;
        const bool linked = fr.linked && nb > 1;
        std::vector<uint64_t> h_in_off, h_slot_off, seg, h_soff;
        std::vector<uint32_t> h_in_len, h_cap, produced, h_first, h_slen;
        std::vector<uint8_t> h_pick;
        std::vector<int32_t> status;
        std::vector<uint64_t> expected;
        for (uint32_t g0 = 0; g0 < nb;) {
            // a group: as many blocks as fit the budget (a linked frame is one dependency chain: one group)
            uint32_t g1 = g0;
            uint64_t slot_total = 0;
            while (g1 < nb) {
                const uint64_t c = blocks[g1].stored ? 0 : block_decoded_cap(blocks[g1].payload_len, bs);
                const uint64_t in_span = blocks[g1].payload_off + blocks[g1].payload_len - blocks[g0].payload_off;
                if (!linked && g1 > g0 && (slot_total + c > ctx->frame_budget || in_span > ctx->frame_budget)) break;
                slot_total += (c + 15) & ~15ull;
                g1++;
            }
            const uint32_t gn = g1 - g0;
            const uint64_t in_lo = blocks[g0].payload_off;
            const uint64_t in_bytes = blocks[g1 - 1].payload_off + blocks[g1 - 1].payload_len - in_lo;
            h_in_off.assign(gn, 0); h_slot_off.assign(gn, 0); h_in_len.assign(gn, 0); h_cap.assign(gn, 0);
            h_pick.assign(gn, 0); produced.assign(gn, 0); status.assign(gn, 0); expected.assign(gn, 0); seg.assign(gn + 1, 0);
            uint64_t so = 0;
            for (uint32_t k = 0; k < gn; k++) {
                const FrameBlockRef &b = blocks[g0 + k];
                h_in_off[k] = b.payload_off - in_lo;
                h_in_len[k] = b.stored ? 0 : b.payload_len;            // stored blocks are only gathered
                h_pick[k] = b.stored ? 1 : 0;
                h_slot_off[k] = so;
                h_cap[k] = b.stored ? 0 : (uint32_t)block_decoded_cap(b.payload_len, bs);
                so += ((uint64_t)h_cap[k] + 15) & ~15ull;
            }
            CTX_CUDA(ctx, ctx->d_in.reserve(in_bytes + 16));
            CTX_CUDA(ctx, ctx->d_slots.reserve(so + 16));
            CTX_CUDA(ctx, ctx->d_in_off.reserve(gn)); CTX_CUDA(ctx, ctx->d_in_len.reserve(gn));
            CTX_CUDA(ctx, ctx->d_out_off.reserve(gn)); CTX_CUDA(ctx, ctx->d_out_cap.reserve(gn));
            CTX_CUDA(ctx, ctx->d_out_len.reserve(gn)); CTX_CUDA(ctx, ctx->d_status.reserve(gn));
            CTX_CUDA(ctx, ctx->d_expected.reserve(gn));
            CTX_CUDA(ctx, ctx->d_pick.reserve(gn)); CTX_CUDA(ctx, ctx->d_seg_off.reserve(gn + 1));
            CTX_CUDA(ctx, ctx->d_payload_len.reserve(gn));
            CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in.p, in + in_lo, in_bytes, cudaMemcpyHostToDevice, s));
            CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_off.p, h_in_off.data(), gn * 8, cudaMemcpyHostToDevice, s));
            CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_in_len.p, h_in_len.data(), gn * 4, cudaMemcpyHostToDevice, s));
            CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_off.p, h_slot_off.data(), gn * 8, cudaMemcpyHostToDevice, s));
            CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_out_cap.p, h_cap.data(), gn * 4, cudaMemcpyHostToDevice, s));
            CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_pick.p, h_pick.data(), gn, cudaMemcpyHostToDevice, s));
            BatchArgs a{ctx->d_in.p, ctx->d_in_off.p, ctx->d_in_len.p, nullptr, ctx->d_slots.p, ctx->d_out_off.p,
                        ctx->d_out_cap.p, ctx->d_out_len.p, ctx->d_status.p, ctx->d_expected.p, gn, nullptr};
            lz4b200_status st;
            if (linked) {
                // BlockMode::Linked (frame/decompress.rs:196-222): the blocks of a frame form a dependency chain; the
                // linked kernel resolves offsets that reach before a block in the outputs of its predecessors
                h_first.assign(gn, 0); h_slen.assign(gn, 0); h_soff.assign(gn, 0);
                for (uint32_t k = 0; k < gn; k++) {
                    h_slen[k] = blocks[g0 + k].stored ? blocks[g0 + k].payload_len : 0;
                    h_soff[k] = h_in_off[k];
                }
                CTX_CUDA(ctx, ctx->d_link_first.reserve(gn)); CTX_CUDA(ctx, ctx->d_stored_len.reserve(gn));
                CTX_CUDA(ctx, ctx->d_stored_off.reserve(gn)); CTX_CUDA(ctx, ctx->d_done.reserve(gn));
                CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_link_first.p, h_first.data(), gn * 4, cudaMemcpyHostToDevice, s));
                CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_stored_len.p, h_slen.data(), gn * 4, cudaMemcpyHostToDevice, s));
                CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_stored_off.p, h_soff.data(), gn * 8, cudaMemcpyHostToDevice, s));
                CTX_CUDA(ctx, cudaMemsetAsync(ctx->d_done.p, 0, gn * 4, s));
                a.link_first = ctx->d_link_first.p; a.stored_off = ctx->d_stored_off.p;
                a.stored_len = ctx->d_stored_len.p; a.done = ctx->d_done.p;
                a.tickets = ctx->d_tickets;
                const uint32_t grid = std::min<uint32_t>((gn + 3) / 4, (uint32_t)ctx->sm_count * 8);
                lz4_decompress_blocks_linked<32><<<grid, 128, 0, s>>>(a);
                st = ctx->check(cudaGetLastError(), "linked decode launch") ? LZ4B200_OK : LZ4B200_CUDA_ERROR;
            } else {
                st = launch_decompress(ctx, a, s);
            }
            if (st != LZ4B200_OK) return st;
            CTX_CUDA(ctx, cudaMemcpyAsync(produced.data(), ctx->d_out_len.p, gn * 4, cudaMemcpyDeviceToHost, s));
            CTX_CUDA(ctx, cudaMemcpyAsync(status.data(), ctx->d_status.p, gn * 4, cudaMemcpyDeviceToHost, s));
            CTX_CUDA(ctx, cudaMemcpyAsync(expected.data(), ctx->d_expected.p, gn * 8, cudaMemcpyDeviceToHost, s));
            CTX_CUDA(ctx, cudaStreamSynchronize(s));

            // first failing block (stream order) wins over anything the walk found later
            uint32_t good = gn;
            for (uint32_t k = 0; k < gn; k++) {
                if (blocks[g0 + k].stored) { produced[k] = blocks[g0 + k].payload_len; status[k] = 0; continue; }
                if (status[k] != 0) { good = k; break; }
            }
            uint64_t gtotal = 0;
            for (uint32_t k = 0; k < good; k++) { seg[k] = gtotal; gtotal += produced[k]; }
            seg[good] = gtotal;
            if (total + gtotal > cap) { *written = total; return LZ4B200_FRAME_OUTPUT_FULL; }
            if (gtotal) {
                CTX_CUDA(ctx, ctx->d_out.reserve(gtotal + 16));
                CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_seg_off.p, seg.data(), (good + 1) * 8, cudaMemcpyHostToDevice, s));
                CTX_CUDA(ctx, cudaMemcpyAsync(ctx->d_payload_len.p, produced.data(), good * 4, cudaMemcpyHostToDevice, s));
                GatherArgs g{ctx->d_slots.p, ctx->d_in.p, ctx->d_out_off.p, ctx->d_in_off.p, ctx->d_payload_len.p,
                             ctx->d_payload_len.p, ctx->d_pick.p, nullptr, ctx->d_out.p, ctx->d_seg_off.p, good};
                gather_segments_kernel<<<std::min<uint32_t>(good, (uint32_t)ctx->sm_count * 8), 256, 0, s>>>(g);
                CTX_CUDA(ctx, cudaGetLastError());
                CTX_CUDA(ctx, cudaMemcpyAsync(out + total, ctx->d_out.p, gtotal, cudaMemcpyDeviceToHost, s));
                CTX_CUDA(ctx, cudaStreamSynchronize(s));
                if (fr.has_checksum) content.update(out + total, gtotal);
            }
            total += gtotal;
            *written = total;
            if (good < gn) {
                if (block_status) *block_status = status[good];
                if (status[good] == LZ4B200_DEC_OUTPUT_TOO_SMALL) {
                    if (err_expected) *err_expected = expected[good];
                    if (err_actual) *err_actual = h_cap[good];
                }
                return LZ4B200_FRAME_DECOMPRESSION_ERROR;
            }
            g0 = g1;
        }
    }
    if (walk_err != LZ4B200_OK) return walk_err;

    // ---- content size / checksum at the EndMark (decompress.rs:312-331) -----------------------------
    if (fr.closed) {
        if (fr.has_size && total != fr.content_size) {
            if (err_expected) *err_expected = fr.content_size;
            if (err_actual) *err_actual = total;
            return LZ4B200_FRAME_CONTENT_LENGTH;
        }
        if (fr.has_checksum && content.digest() != fr.content_checksum) return LZ4B200_FRAME_CONTENT_CHECKSUM;
    }
    return LZ4B200_OK;
}

// Every concatenated frame of `in`, back to back (a convenience over lz4b200_frame_decompress_next: the reference's
// reader stops at each EndMark, frame/decompress.rs:310-331, and a caller that cares about frame boundaries uses _next).
lz4b200_status lz4b200_frame_decompress(lz4b200_ctx *ctx, const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                        size_t *written, int *block_status)
{
    if (!ctx || !written || (!in && n) || (!out && cap)) return LZ4B200_INVALID_ARGUMENT;
    *written = 0;
    if (block_status) *block_status = 0;
    size_t ip = 0;
    while (ip < n) {
        size_t used = 0, w = 0;
        const lz4b200_status st = lz4b200_frame_decompress_next(ctx, in + ip, n - ip, out + *written, cap - *written, &used,
                                                                &w, block_status, nullptr, nullptr);
        *written += w;
        if (st != LZ4B200_OK) return st;
        if (used == 0) break;
        ip += used;
    }
    return LZ4B200_OK;
}

}  // extern "C"
