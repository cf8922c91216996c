/*
 * linked_frame_ref.c — CPU restatement of lz4_flex's FrameEncoder with BlockMode::Linked (frame/compress.rs:261-371,
 * block/compress.rs:318-489), the parity reference of the linked batch frame encoder.  Test infrastructure only:
 * nothing in the product links or runs this.  tests/linked_ref.py builds it with gcc and calls it through ctypes.
 *
 * It stands apart from the C oracle (oracle/lz4_oracle.c), whose independent-block parse it shares in design: a u32
 * table of 4 096 slots, the 5-byte hash, the probe loop with its growing step, backward and forward extension, and the
 * cur - 2 re-insert.  What linked blocks add, modelled here the way the encoder keeps its buffer:
 *   - one table for the whole frame, zeroed when the frame opens and carried from block to block;
 *   - a buffer of 2 * bs + 64 KiB.  Its head holds the block and the blocks before it (the prefix, input_pos bytes);
 *     an ext_dict of up to 64 KiB of older bytes lies elsewhere in it.  src_start / src_end / ext_off / ext_len /
 *     stream move exactly as in write_block (:323-356), and each block is parsed as
 *     compress_internal(src[..src_end], src_start, ext_dict, stream);
 *   - a candidate at or after `stream` is in the input (prefix or block) and extends like any in-input match; one
 *     below it is in the ext_dict, extends backwards to the ext_dict's first byte and forwards to its last;
 *   - position 0 goes into the table before the parse only when input_pos == 0 and stream == 0 (:353-359);
 *   - before each block, when stream + bs + 64 KiB >= 2^31 - 1, every entry drops by stream - ext_len (saturating)
 *     and stream becomes ext_len (:266-271).
 * Blocks are cut as FrameEncoder cuts them: full blocks of bs from write_all, the rest at a flush or at finish.
 * `flush_every` > 0 models write_all(chunk of flush_every bytes) + flush() in a loop.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MINMATCH 4u
#define MFLIMIT 12u
#define END_OFFSET 6u
#define MIN_LENGTH 13u
#define MAX_DISTANCE 65535u
#define SLOTS 4096u
#define WINDOW 65536u

static inline uint32_t ld32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static inline uint64_t ld64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline void st32(uint8_t *p, uint32_t v) { memcpy(p, &v, 4); }

static inline uint32_t slot5(const uint8_t *p) { return (uint32_t)((((ld64(p) << 24) * 889523592379ULL) >> 48) >> 4); }

static size_t max_output(size_t n) { return 16 + 4 + (size_t)((uint64_t)n * 110 / 100); }

static uint8_t *put_len(uint8_t *op, size_t v)            /* length-extension bytes of v = len - 15 */
{
    while (v >= 255) { *op++ = 255; v -= 255; }
    *op++ = (uint8_t)v;
    return op;
}

static uint8_t *last_literals(uint8_t *op, const uint8_t *from, size_t len)
{
    *op++ = (uint8_t)((len < 15 ? len : 15) << 4);
    if (len >= 15) op = put_len(op, len - 15);
    memcpy(op, from, len);
    return op + len;
}

/* One block: in[pos, n) with the prefix in[0, pos), the ext_dict dict[0, dlen) ending at stream offset `off`. */
static size_t encode_block(const uint8_t *in, size_t pos, size_t n, uint8_t *out, uint32_t *tab, size_t off,
                           const uint8_t *dict, size_t dlen)
{
    uint8_t *op = out;
    if (n - pos < MIN_LENGTH) return (size_t)(last_literals(op, in + pos, n - pos) - out);
    const size_t last_probe = n - MFLIMIT, lim = n - END_OFFSET, dict_off = off - dlen;
    size_t anchor = pos, cur = pos;
    if (pos == 0 && off == 0) { tab[slot5(in)] = 0; cur = 1; }
    for (;;) {
        size_t misses = 32, next = cur, cand, clen;
        const uint8_t *csrc;
        uint32_t dist;
        for (;;) {
            const size_t step = misses >> 5;
            misses++;
            cur = next; next += step;
            if (cur > last_probe) return (size_t)(last_literals(op, in + anchor, n - anchor) - out);
            const uint32_t s = slot5(in + cur);
            cand = tab[s];
            tab[s] = (uint32_t)(cur + off);
            if (off + cur - cand > MAX_DISTANCE) continue;
            dist = (uint32_t)(off + cur - cand);
            if (cand >= off) { cand -= off; csrc = in; clen = n; }
            else if (dlen) { cand -= dict_off; csrc = dict; clen = dlen; }
            else continue;                                  /* before the input, and no ext_dict */
            if (ld32(csrc + cand) == ld32(in + cur)) break;
        }
        while (cand > 0 && cur > anchor && in[cur - 1] == csrc[cand - 1]) { cur--; cand--; }
        const size_t lit = cur - anchor;
        cur += MINMATCH; cand += MINMATCH;
        size_t extra = 0;                                   /* limited by n - END_OFFSET and by the source's end */
        while (cur + extra < lim && cand + extra < clen && in[cur + extra] == csrc[cand + extra]) extra++;
        cur += extra;
        tab[slot5(in + cur - 2)] = (uint32_t)(cur - 2 + off);
        *op++ = (uint8_t)(((lit < 15 ? lit : 15) << 4) | (extra < 15 ? extra : 15));
        if (lit >= 15) op = put_len(op, lit - 15);
        memcpy(op, in + anchor, lit); op += lit;
        *op++ = (uint8_t)dist; *op++ = (uint8_t)(dist >> 8);
        if (extra >= 15) op = put_len(op, extra - 15);
        anchor = cur;
    }
}

/* XXH32 (twox-hash XxHash32), one-shot and streaming */
#define P1 2654435761u
#define P2 2246822519u
#define P3 3266489917u
#define P4 668265263u
#define P5 374761393u
static inline uint32_t rotl(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
static inline uint32_t rnd(uint32_t a, uint32_t v) { return rotl(a + v * P2, 13) * P1; }

typedef struct { uint32_t acc[4]; uint8_t buf[16]; uint32_t fill; uint64_t total; } xxh;

static void xxh_init(xxh *s)
{
    s->acc[0] = P1 + P2; s->acc[1] = P2; s->acc[2] = 0; s->acc[3] = 0u - P1;
    s->fill = 0; s->total = 0;
}
static void xxh_update(xxh *s, const uint8_t *p, size_t n)
{
    s->total += n;
    while (n) {
        size_t take = 16 - s->fill < n ? 16 - s->fill : n;
        memcpy(s->buf + s->fill, p, take);
        s->fill += (uint32_t)take; p += take; n -= take;
        if (s->fill == 16) {
            for (int i = 0; i < 4; i++) s->acc[i] = rnd(s->acc[i], ld32(s->buf + 4 * i));
            s->fill = 0;
        }
    }
}
static uint32_t xxh_digest(const xxh *s)
{
    uint32_t h = s->total >= 16 ? rotl(s->acc[0], 1) + rotl(s->acc[1], 7) + rotl(s->acc[2], 12) + rotl(s->acc[3], 18)
                                : P5;
    h += (uint32_t)s->total;
    const uint8_t *p = s->buf, *e = s->buf + s->fill;
    for (; p + 4 <= e; p += 4) h = rotl(h + ld32(p) * P3, 17) * P4;
    for (; p < e; p++) h = rotl(h + (*p) * P5, 11) * P1;
    h ^= h >> 15; h *= P2; h ^= h >> 13; h *= P3; h ^= h >> 16;
    return h;
}
static uint32_t xxh32(const uint8_t *p, size_t n) { xxh s; xxh_init(&s); xxh_update(&s, p, n); return xxh_digest(&s); }

/* flags: 1 block checksums, 2 content checksum, 4 content size.  block_size_id 0 = Auto (from the first write). */
size_t lfr_frame_bound(size_t n, int block_size_id, size_t flush_every)
{
    (void)block_size_id;
    return 19 + n + 8 * (n / 1024 + 2) + (flush_every ? 8 * (n / flush_every + 2) : 0) + 8;
}

int64_t lfr_frame_compress(const uint8_t *in, size_t n, int block_size_id, unsigned flags, size_t flush_every,
                           uint8_t *out, size_t cap)
{
    if (block_size_id == 0) {
        const size_t first = flush_every && flush_every < n ? flush_every : n;
        block_size_id = first > (256u << 10) ? 7 : first > (64u << 10) ? 5 : 4;
    }
    if (block_size_id < 4 || block_size_id > 7) return -2;
    const size_t bs = (size_t)64 << (10 + 2 * (block_size_id - 4));
    if (cap < lfr_frame_bound(n, block_size_id, flush_every)) return -1;

    uint8_t *op = out;                                      /* header (header.rs:232-275), the 0x20 flag clear */
    st32(op, 0x184D2204u);
    uint8_t flg = 0x40;
    if (flags & 1) flg |= 0x10;
    if (flags & 2) flg |= 0x04;
    if (flags & 4) flg |= 0x08;
    op[4] = flg;
    op[5] = (uint8_t)(block_size_id << 4);
    size_t h = 6;
    if (flags & 4) { uint64_t cs = n; memcpy(op + h, &cs, 8); h += 8; }
    op[h] = (uint8_t)(xxh32(op + 4, h - 4) >> 8);
    op += h + 1;

    uint32_t *tab = (uint32_t *)calloc(SLOTS, sizeof(uint32_t));
    uint8_t *scratch = (uint8_t *)malloc(max_output(bs));
    uint8_t *src = (uint8_t *)malloc(2 * bs + WINDOW);
    xxh content; xxh_init(&content);
    size_t src_start = 0, src_end = 0, ext_off = 0, ext_len = 0, stream = 0, pos = 0, since_flush = 0;
    while (pos < n) {
        size_t len = n - pos < bs ? n - pos : bs;
        if (flush_every && flush_every - since_flush < len) len = flush_every - since_flush;
        memcpy(src + src_end, in + pos, len);
        src_end += len;
        if (stream + bs + WINDOW >= 0x7FFFFFFFu) {          /* :266-271 */
            const size_t shift = stream - ext_len;
            for (unsigned i = 0; i < SLOTS; i++) tab[i] = tab[i] > shift ? tab[i] - (uint32_t)shift : 0;
            stream = ext_len;
        }
        size_t c = encode_block(src, src_start, src_end, scratch, tab, stream, ext_len ? src + ext_off : NULL, ext_len);
        const uint8_t *payload = scratch;
        uint32_t info = (uint32_t)c;
        if (c >= len) { payload = in + pos; info = (uint32_t)len | 0x80000000u; c = len; }   /* :301-306 */
        st32(op, info); op += 4;
        memcpy(op, payload, c); op += c;
        if (flags & 1) { st32(op, xxh32(payload, c)); op += 4; }
        if (flags & 2) xxh_update(&content, in + pos, len);
        src_start += len;                                   /* :323-356 */
        if (src_start >= bs + WINDOW) {
            ext_off = src_end - WINDOW;
            ext_len = WINDOW;
            stream += src_end;
            src_start = src_end = 0;
        } else if (src_start + ext_len > WINDOW) {
            size_t delta = src_start + ext_len - WINDOW;
            if (delta > ext_len) delta = ext_len;
            ext_off += delta;
            ext_len -= delta;
        }
        pos += len; since_flush += len;
        if (flush_every && since_flush == flush_every) since_flush = 0;
    }
    st32(op, 0); op += 4;
    if (flags & 2) { st32(op, xxh_digest(&content)); op += 4; }
    free(tab); free(scratch); free(src);
    return op - out;
}
