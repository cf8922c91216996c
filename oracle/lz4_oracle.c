/*
 * lz4_oracle.c — CPU restatement of lz4_flex's LZ4 block codec and frame container.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is the parity checker for the CUDA path and
 * the CPU baseline of bench.py.  Nothing under lz4_flex_b200/ may include, link or
 * call it; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs do.
 *
 * Provenance: lz4_flex is Rust and no Rust toolchain exists in the build image, so the
 * reference cannot be compiled here.  This is an independent C restatement of the
 * algorithm (not a transliteration), pinned against
 *   - every hand-written decode vector + error variant of the reference's unit tests
 *     (src/block/decompress.rs:535-621, same set in decompress_safe.rs:397-483),
 *   - the reference's ratio bounds (tests/tests.rs:158-192),
 *   - the conformant-last-block test (src/block/compress.rs:952-988),
 *   - the frame header known bytes (fuzz/fuzz_targets/fuzz_decomp_corrupt_frame.rs:26-27),
 *   - the legacy-frame fixture benches/dickens.lz4 (tests/tests.rs:741-745),
 *   - cross-decoding by the system liblz4 1.9.4 (the reference's own interop check,
 *     tests/tests.rs:109-147), including LZ4_decompress_safe_usingDict for the dictionary
 *     encoder and LZ4F-written linked-block frames for the frame decoder,
 *   - the reference's dictionary unit tests (src/block/compress.rs:892-950,
 *     src/block/decompress.rs:593-601).
 * COMPRESSED BYTES are not pinned by any reference fixture ("parity unpinned" for the
 * exact encoder output; see DESIGN.md §oracle): the known-answers in tests/golden/ come
 * from two independent restatements agreeing (this file and the surveyor's), not from
 * lz4_flex itself.
 *
 * What follows what (reference file:line, relative to the lz4_flex v0.12.0 source tree):
 *   slot4()/slot5()          src/block/hashtable.rs:19-21, 27-34, 77-83, 121-127
 *   lz4o_max_output_size()   src/block/compress.rs:588-590
 *   encode_* (core parse)    src/block/compress.rs:318-489  (helpers :65-96, :156-247, :272-287)
 *   lz4o_compress_block()    src/block/compress.rs:554-567  (table/hash choice), :599
 *   lz4o_decompress_block()  src/block/decompress.rs:201-449 (error order), cross-read with
 *                            src/block/decompress_safe.rs:93-247
 *   lz4o_compress_block_dict()   src/block/compress.rs:554-583 (table choice, init_dict), :412-421 (ext_dict
 *                            candidates), :156-216 / :272-287 (extension confined to the candidate's source)
 *   lz4o_decompress_block_dict() src/block/decompress.rs:85-109 (copy_from_dict), :287-301, :399-427
 *   linked frames (decode)   src/frame/decompress.rs:196-222, 277-305
 *   lz4o_xxh32()             twox-hash 2.x XxHash32 (Cargo.toml:51) = standard XXH32
 *   lz4o_frame_*()           src/frame/header.rs:232-372, :383-410;
 *                            src/frame/compress.rs:234-371; src/frame/decompress.rs:109-342
 */
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <stdlib.h>

#include "lz4_oracle.h"

/* ------------------------------------------------------------------------------------------ */
/* little helpers                                                                              */

static inline uint32_t ld32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }
static inline uint64_t ld64(const uint8_t *p) { uint64_t v; memcpy(&v, p, 8); return v; }
static inline void st16(uint8_t *p, uint16_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); }
static inline void st32(uint8_t *p, uint32_t v) { memcpy(p, &v, 4); }

#define LZ4O_MINMATCH      4u
#define LZ4O_MFLIMIT       12u     /* block/mod.rs:46 */
#define LZ4O_END_OFFSET    6u      /* block/mod.rs:55: LAST_LITERALS + 1 */
#define LZ4O_MIN_LENGTH    13u     /* block/mod.rs:61 */
#define LZ4O_MAX_DISTANCE  65535u  /* block/mod.rs:64 */
#define LZ4O_SLOTS         4096u
#define LZ4O_WINDOW        65536u  /* block/mod.rs: WINDOW_SIZE */

/* 12-bit slot of the 4-byte multiplicative hash (u16 table, inputs < 65535 bytes). */
static inline uint32_t slot4(const uint8_t *p)
{
    return ((ld32(p) * 2654435761u) >> 16) >> 4;
}
/* 12-bit slot of the 5-byte hash: low five bytes of an 8-byte little-endian load. */
static inline uint32_t slot5(const uint8_t *p)
{
    return (uint32_t)((((ld64(p) << 24) * 889523592379ULL) >> 48) >> 4);
}

size_t lz4o_max_output_size(size_t n)
{
    return 16 + 4 + (size_t)((uint64_t)n * 110 / 100);
}

/* Length-extension bytes: v = len - 15. */
static inline uint8_t *put_ext(uint8_t *op, size_t v)
{
    while (v >= 255) { *op++ = 255; v -= 255; }
    *op++ = (uint8_t)v;
    return op;
}

static inline uint8_t *put_tail_literals(uint8_t *op, const uint8_t *in, size_t from, size_t n)
{
    size_t len = n - from;
    *op++ = (uint8_t)((len < 15 ? len : 15) << 4);
    if (len >= 15) op = put_ext(op, len - 15);
    memcpy(op, in + from, len);
    return op + len;
}

/* Forward match length from (cur, cand), cur limited to n - END_OFFSET. */
static inline size_t common_prefix(const uint8_t *in, size_t cur, size_t cand, size_t n)
{
    size_t lim = n - LZ4O_END_OFFSET, start = cur;
    if (cur >= lim) return 0;
    while (cur + 8 <= lim) {
        uint64_t x = ld64(in + cur) ^ ld64(in + cand);
        if (x) return cur - start + (size_t)(__builtin_ctzll(x) >> 3);
        cur += 8; cand += 8;
    }
    while (cur < lim && in[cur] == in[cand]) { cur++; cand++; }
    return cur - start;
}

/* Forward match length against an external source (the dictionary): limited by the input's
 * n - END_OFFSET and by the end of the source (compress.rs:156-216, max_candidate_match). */
static inline size_t common_prefix_ext(const uint8_t *in, size_t cur, size_t n, const uint8_t *src, size_t cand,
                                       size_t srclen)
{
    size_t lim = n - LZ4O_END_OFFSET, k = 0;
    if (cur >= lim) return 0;
    size_t room = lim - cur;
    if (srclen - cand < room) room = srclen - cand;
    while (k < room && in[cur + k] == src[cand + k]) k++;
    return k;
}

/*
 * One parse, two table layouts.  TAB_T/SLOT are the only differences between the
 * "small input" (u16 + hash4) and the general (u32 + hash5) encoders.
 * `off` is input_stream_offset; `dict`/`dlen` the external dictionary that logically precedes the input
 * (ext_dict of compress_internal, compress.rs:318-489; dlen == 0: USE_DICT = false).
 */
#define DEFINE_ENCODER(NAME, TAB_T, SLOT)                                                        \
static int64_t NAME(const uint8_t *in, size_t n, uint8_t *out, size_t cap,                       \
                    TAB_T *tab, size_t off, const uint8_t *dict, size_t dlen)                    \
{                                                                                                \
    if (cap < lz4o_max_output_size(n)) return -1;            /* CompressError::OutputTooSmall */ \
    uint8_t *op = out;                                                                           \
    if (n < LZ4O_MIN_LENGTH) return put_tail_literals(op, in, 0, n) - out;                       \
    const size_t last_probe = n - LZ4O_MFLIMIT;                                                  \
    const size_t dict_off = off - dlen;                      /* ext_dict_stream_offset */        \
    size_t anchor = 0, cur = 0;                                                                  \
    if (off == 0) { tab[SLOT(in)] = 0; cur = 1; }   /* a block may not start with a match */     \
    for (;;) {                                                                                   \
        size_t misses = 32, next = cur, cand;                                                    \
        uint32_t dist;                                                                           \
        const uint8_t *csrc;                                                                     \
        size_t clen;                                                                             \
        for (;;) {                                                                               \
            size_t step = misses >> 5; misses++;                                                 \
            cur = next; next += step;                                                            \
            if (cur > last_probe) return put_tail_literals(op, in, anchor, n) - out;             \
            uint32_t s = SLOT(in + cur);                                                         \
            cand = tab[s];                                                                       \
            tab[s] = (TAB_T)(cur + off);                                                         \
            if (off + cur - cand > LZ4O_MAX_DISTANCE) continue;                                  \
            dist = (uint32_t)(off + cur - cand);                                                 \
            if (cand >= off) { cand -= off; csrc = in; clen = n; }                               \
            else if (dlen) { cand -= dict_off; csrc = dict; clen = dlen; }                       \
            else continue;                        /* entry left by an earlier frame block */     \
            if (ld32(csrc + cand) == ld32(in + cur)) break;                                      \
        }                                                                                        \
        while (cand > 0 && cur > anchor && in[cur - 1] == csrc[cand - 1]) { cur--; cand--; }     \
        size_t lit = cur - anchor;                                                               \
        cur += LZ4O_MINMATCH; cand += LZ4O_MINMATCH;                                             \
        size_t extra = csrc == in ? common_prefix(in, cur, cand, n)                              \
                                  : common_prefix_ext(in, cur, n, csrc, cand, clen);             \
        cur += extra;                                                                            \
        tab[SLOT(in + cur - 2)] = (TAB_T)(cur - 2 + off);                                        \
        *op++ = (uint8_t)(((lit < 15 ? lit : 15) << 4) | (extra < 15 ? extra : 15));             \
        if (lit >= 15) op = put_ext(op, lit - 15);                                               \
        memcpy(op, in + anchor, lit); op += lit;                                                 \
        st16(op, (uint16_t)dist); op += 2;                                                       \
        if (extra >= 15) op = put_ext(op, extra - 15);                                           \
        anchor = cur;                                                                            \
    }                                                                                            \
}

DEFINE_ENCODER(encode_u16_h4, uint16_t, slot4)
DEFINE_ENCODER(encode_u32_h5, uint32_t, slot5)

int64_t lz4o_compress_block(const uint8_t *in, size_t n, uint8_t *out, size_t cap)
{
    if (n < 65535) {
        uint16_t tab[LZ4O_SLOTS];
        memset(tab, 0, sizeof tab);
        return encode_u16_h4(in, n, out, cap, tab, 0, NULL, 0);
    } else {
        uint32_t *tab = (uint32_t *)calloc(LZ4O_SLOTS, sizeof(uint32_t));
        int64_t r = encode_u32_h5(in, n, out, cap, tab, 0, NULL, 0);
        free(tab);
        return r;
    }
}

int64_t lz4o_compress_block_with_table(const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                       uint32_t *table4096, uint64_t stream_offset)
{
    return encode_u32_h5(in, n, out, cap, table4096, (size_t)stream_offset, NULL, 0);
}

/* compress_into_with_dict (compress.rs:554-583, 610-616): the dictionary is cut to its last 64 KiB, every third
 * position with 8 readable bytes is put into the table (init_dict), the table layout follows dict + input length,
 * and the input is parsed at stream offset = dictionary length.  Dictionaries of <= 3 bytes are dropped
 * (compress_into_vec_with_dict, compress.rs:626-628; the slice API would read past a shorter one). */
int64_t lz4o_compress_block_dict(const uint8_t *in, size_t n, const uint8_t *dict, size_t dlen, uint8_t *out,
                                 size_t cap)
{
    if (dlen <= 3) { dict = NULL; dlen = 0; }
    if (dlen > LZ4O_WINDOW) { dict += dlen - LZ4O_WINDOW; dlen = LZ4O_WINDOW; }
    if (dlen + n < 65535) {
        uint16_t tab[LZ4O_SLOTS];
        memset(tab, 0, sizeof tab);
        for (size_t i = 0; i + 8 <= dlen; i += 3) tab[slot4(dict + i)] = (uint16_t)i;
        return encode_u16_h4(in, n, out, cap, tab, dlen, dict, dlen);
    } else {
        uint32_t *tab = (uint32_t *)calloc(LZ4O_SLOTS, sizeof(uint32_t));
        for (size_t i = 0; i + 8 <= dlen; i += 3) tab[slot5(dict + i)] = (uint32_t)i;
        int64_t r = encode_u32_h5(in, n, out, cap, tab, dlen, dict, dlen);
        free(tab);
        return r;
    }
}

int64_t lz4o_compress_prepend_size(const uint8_t *in, size_t n, uint8_t *out, size_t cap)
{
    if (cap < 4) return -1;
    st32(out, (uint32_t)n);
    int64_t r = lz4o_compress_block(in, n, out + 4, cap - 4);
    return r < 0 ? r : r + 4;
}

/* ------------------------------------------------------------------------------------------ */
/* block decoder                                                                               */

/* Reads 255-run length bytes; returns 0 on success, nonzero when the input runs out. */
static inline int get_ext(const uint8_t *in, size_t n, size_t *ip, size_t *len)
{
    for (;;) {
        if (*ip >= n) return 1;
        uint8_t b = in[(*ip)++];
        *len += b;
        if (b != 255) return 0;
    }
}

/* out[op .. op+mlen) = the bytes `dist` back in the virtual buffer [dict | out] (copy_from_dict + duplicate,
 * decompress.rs:85-109, 292-301, 410-427): byte-serial LZ77 semantics across the dictionary/output seam. */
static inline void copy_match_dict(uint8_t *out, size_t op, size_t dist, size_t mlen, const uint8_t *dict, size_t dlen)
{
    for (size_t i = 0; i < mlen; i++) {
        size_t at = op + i;
        out[at] = at >= dist ? out[at - dist] : dict[dlen + at - dist];
    }
}

int lz4o_decompress_block_dict(const uint8_t *in, size_t n, const uint8_t *dict, size_t dlen, uint8_t *out,
                               size_t cap, size_t *written, size_t *err_expected, size_t *err_actual)
{
    size_t ip = 0, op = 0;
    *written = 0;
    if (n == 0) return LZ4O_ERR_EXPECTED_ANOTHER_BYTE;
    for (;;) {
        uint8_t tok = in[ip++];
        size_t lit = tok >> 4, mlen = (tok & 15) + LZ4O_MINMATCH;

        /* Short-sequence fast path: identical results, only taken when no check can fire
         * except the two offset checks. */
        if (lit != 15 && mlen != 19 && n - ip >= 19 && cap - op > 34) {
            memcpy(out + op, in + ip, 16);
            ip += lit; op += lit;
            size_t dist = (size_t)in[ip] | ((size_t)in[ip + 1] << 8);
            ip += 2;
            if (dist == 0) return LZ4O_ERR_OFFSET_ZERO;
            if (dist > op + dlen) return LZ4O_ERR_OFFSET_OOB;
            if (dist > op) copy_match_dict(out, op, dist, mlen, dict, dlen);
            else if (dist >= 18) memcpy(out + op, out + op - dist, 18);
            else for (size_t i = 0; i < mlen; i++) out[op + i] = out[op - dist + i];
            op += mlen;
            continue;
        }

        if (lit) {
            if (lit == 15 && get_ext(in, n, &ip, &lit)) return LZ4O_ERR_EXPECTED_ANOTHER_BYTE;
            if (lit > n - ip) return LZ4O_ERR_LITERAL_OOB;
            if (lit > cap - op) {
                *err_expected = op + lit; *err_actual = cap;
                return LZ4O_ERR_OUTPUT_TOO_SMALL;
            }
            memcpy(out + op, in + ip, lit);
            ip += lit; op += lit;
        }
        if (ip >= n) break;                                  /* a block ends after literals */
        if (n - ip < 2) return LZ4O_ERR_EXPECTED_ANOTHER_BYTE;
        size_t dist = (size_t)in[ip] | ((size_t)in[ip + 1] << 8);
        ip += 2;
        if (dist == 0) return LZ4O_ERR_OFFSET_ZERO;
        if (mlen == 19 && get_ext(in, n, &ip, &mlen)) return LZ4O_ERR_EXPECTED_ANOTHER_BYTE;
        if (dist > op + dlen) return LZ4O_ERR_OFFSET_OOB;
        if (mlen > cap - op) {
            *err_expected = op + mlen; *err_actual = cap;
            return LZ4O_ERR_OUTPUT_TOO_SMALL;
        }
        if (dist > op) {
            copy_match_dict(out, op, dist, mlen, dict, dlen);
        } else if (dist >= mlen) {
            memcpy(out + op, out + op - dist, mlen);
        } else if (dist == 1) {
            memset(out + op, out[op - 1], mlen);
        } else {
            for (size_t i = 0; i < mlen; i++) out[op + i] = out[op - dist + i];
        }
        op += mlen;
        if (ip >= n) return LZ4O_ERR_EXPECTED_ANOTHER_BYTE;  /* may not end on a match */
    }
    *written = op;
    return LZ4O_OK;
}

int lz4o_decompress_block(const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                          size_t *written, size_t *err_expected, size_t *err_actual)
{
    return lz4o_decompress_block_dict(in, n, NULL, 0, out, cap, written, err_expected, err_actual);
}

int lz4o_decompress_size_prepended(const uint8_t *in, size_t n, uint8_t *out, size_t cap,
                                   size_t *written, size_t *err_expected, size_t *err_actual)
{
    *written = 0;
    if (n < 4) return LZ4O_ERR_EXPECTED_ANOTHER_BYTE;           /* block/mod.rs:151-157 */
    size_t want = ld32(in);
    if (want < cap) cap = want;       /* the reference allocates exactly the prefixed size */
    return lz4o_decompress_block(in + 4, n - 4, out, cap, written, err_expected, err_actual);
}

/* ------------------------------------------------------------------------------------------ */
/* XXH32                                                                                       */

#define XP1 2654435761u
#define XP2 2246822519u
#define XP3 3266489917u
#define XP4 668265263u
#define XP5 374761393u
static inline uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }
static inline uint32_t xround(uint32_t acc, uint32_t v) { return rotl32(acc + v * XP2, 13) * XP1; }

uint32_t lz4o_xxh32(const uint8_t *p, size_t n, uint32_t seed)
{
    const uint8_t *end = p + n;
    uint32_t h;
    if (n >= 16) {
        uint32_t a = seed + XP1 + XP2, b = seed + XP2, c = seed, d = seed - XP1;
        const uint8_t *lim = end - 16;
        do {
            a = xround(a, ld32(p)); b = xround(b, ld32(p + 4));
            c = xround(c, ld32(p + 8)); d = xround(d, ld32(p + 12));
            p += 16;
        } while (p <= lim);
        h = rotl32(a, 1) + rotl32(b, 7) + rotl32(c, 12) + rotl32(d, 18);
    } else {
        h = seed + XP5;
    }
    h += (uint32_t)n;
    while (p + 4 <= end) { h = rotl32(h + ld32(p) * XP3, 17) * XP4; p += 4; }
    while (p < end) { h = rotl32(h + (*p) * XP5, 11) * XP1; p++; }
    h ^= h >> 15; h *= XP2; h ^= h >> 13; h *= XP3; h ^= h >> 16;
    return h;
}

/* Streaming XXH32 for the content checksum (whole-stream hash fed block by block). */
typedef struct { uint32_t acc[4]; uint8_t buf[16]; uint32_t fill; uint64_t total; uint32_t seed; } xxh32_state;

static void xs_init(xxh32_state *s, uint32_t seed)
{
    s->acc[0] = seed + XP1 + XP2; s->acc[1] = seed + XP2; s->acc[2] = seed; s->acc[3] = seed - XP1;
    s->fill = 0; s->total = 0; s->seed = seed;
}
static void xs_update(xxh32_state *s, const uint8_t *p, size_t n)
{
    s->total += n;
    if (s->fill) {
        size_t take = 16 - s->fill; if (take > n) take = n;
        memcpy(s->buf + s->fill, p, take); s->fill += (uint32_t)take; p += take; n -= take;
        if (s->fill < 16) return;
        for (int i = 0; i < 4; i++) s->acc[i] = xround(s->acc[i], ld32(s->buf + 4 * i));
        s->fill = 0;
    }
    while (n >= 16) {
        for (int i = 0; i < 4; i++) s->acc[i] = xround(s->acc[i], ld32(p + 4 * i));
        p += 16; n -= 16;
    }
    if (n) { memcpy(s->buf, p, n); s->fill = (uint32_t)n; }
}
static uint32_t xs_digest(const xxh32_state *s)
{
    uint32_t h = s->total >= 16
        ? rotl32(s->acc[0], 1) + rotl32(s->acc[1], 7) + rotl32(s->acc[2], 12) + rotl32(s->acc[3], 18)
        : s->seed + XP5;
    h += (uint32_t)s->total;
    const uint8_t *p = s->buf, *end = s->buf + s->fill;
    while (p + 4 <= end) { h = rotl32(h + ld32(p) * XP3, 17) * XP4; p += 4; }
    while (p < end) { h = rotl32(h + (*p) * XP5, 11) * XP1; p++; }
    h ^= h >> 15; h *= XP2; h ^= h >> 13; h *= XP3; h ^= h >> 16;
    return h;
}

/* ------------------------------------------------------------------------------------------ */
/* frame container (independent blocks)                                                        */

#define F_MAGIC        0x184D2204u
#define F_LEGACY_MAGIC 0x184C2102u
#define F_SKIP_LO      0x184D2A50u
#define F_SKIP_HI      0x184D2A5Fu

size_t lz4o_block_size_bytes(int id)
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

int lz4o_auto_block_size_id(size_t first_write_len)
{
    if (first_write_len > (256u << 10)) return 7;
    if (first_write_len > (64u << 10)) return 5;
    return 4;
}

size_t lz4o_frame_header(uint8_t *out, int block_size_id, unsigned flags, uint64_t content_size)
{
    size_t o = 0;
    st32(out, F_MAGIC); o = 4;
    uint8_t flg = 0x40;
    if (flags & LZ4O_F_BLOCK_CHECKSUMS) flg |= 0x10;
    if (flags & LZ4O_F_CONTENT_CHECKSUM) flg |= 0x04;
    if (!(flags & LZ4O_F_LINKED)) flg |= 0x20;
    if (flags & LZ4O_F_CONTENT_SIZE) flg |= 0x08;
    out[o++] = flg;
    out[o++] = (uint8_t)(block_size_id << 4);
    if (flags & LZ4O_F_CONTENT_SIZE) { memcpy(out + o, &content_size, 8); o += 8; }
    out[o] = (uint8_t)(lz4o_xxh32(out + 4, o - 4, 0) >> 8);
    return o + 1;
}

size_t lz4o_frame_bound(size_t n, int block_size_id)
{
    size_t bs = lz4o_block_size_bytes(block_size_id);
    size_t nb = bs ? (n + bs - 1) / bs : 0;
    return 19 + n + nb * 8 + 4 + 4;
}

/*
 * Equivalent of: FrameEncoder::with_frame_info(info, Vec::new()); enc.write_all(in); enc.finish().
 * `flush_every` > 0 instead models write_all(chunk of flush_every bytes) + flush() in a loop,
 * which produces short blocks and shifts the stream-offset phase exactly like the reference.
 */
int64_t lz4o_frame_compress(const uint8_t *in, size_t n, int block_size_id, unsigned flags,
                            size_t flush_every, uint8_t *out, size_t cap)
{
    if (flags & LZ4O_F_LINKED) return -2;                       /* out of scope */
    if (block_size_id == 0) block_size_id = lz4o_auto_block_size_id(flush_every ? (flush_every < n ? flush_every : n) : n);
    const size_t bs = lz4o_block_size_bytes(block_size_id);
    if (!bs || block_size_id == 8) return -2;
    if (cap < lz4o_frame_bound(n, block_size_id) + (flush_every ? 8 * (n / flush_every + 1) : 0)) return -1;

    uint32_t *tab = (uint32_t *)calloc(LZ4O_SLOTS, sizeof(uint32_t));
    uint8_t *scratch = (uint8_t *)malloc(lz4o_max_output_size(bs));
    uint8_t *op = out;
    op += lz4o_frame_header(op, block_size_id, flags, (uint64_t)n);
    xxh32_state content; xs_init(&content, 0);
    size_t off = 0, pos = 0, since_flush = 0;
    while (pos < n) {
        size_t len = n - pos < bs ? n - pos : bs;
        if (flush_every && flush_every - since_flush < len) len = flush_every - since_flush;
        /* frame/compress.rs:266-271: table reposition when the stream offset nears 2^31 */
        if (off + bs + 65536 >= 0x7FFFFFFFu) {
            for (unsigned i = 0; i < LZ4O_SLOTS; i++) tab[i] = tab[i] > off ? tab[i] - (uint32_t)off : 0;
            off = 0;
        }
        int64_t c = encode_u32_h5(in + pos, len, scratch, lz4o_max_output_size(len), tab, off, NULL, 0);
        const uint8_t *payload; uint32_t info;
        if ((size_t)c < len) { payload = scratch; info = (uint32_t)c; }
        else { payload = in + pos; info = (uint32_t)len | 0x80000000u; c = (int64_t)len; }
        st32(op, info); op += 4;
        memcpy(op, payload, (size_t)c); op += c;
        if (flags & LZ4O_F_BLOCK_CHECKSUMS) { st32(op, lz4o_xxh32(payload, (size_t)c, 0)); op += 4; }
        if (flags & LZ4O_F_CONTENT_CHECKSUM) xs_update(&content, in + pos, len);
        off += len; pos += len; since_flush += len;
        if (flush_every && since_flush == flush_every) since_flush = 0;
    }
    st32(op, 0); op += 4;
    if (flags & LZ4O_F_CONTENT_CHECKSUM) { st32(op, xs_digest(&content)); op += 4; }
    free(tab); free(scratch);
    return op - out;
}

/* Decodes every concatenated frame in `in`.  Errors are the LZ4O_FERR_* codes. */
int lz4o_frame_decompress(const uint8_t *in, size_t n, uint8_t *out, size_t cap, size_t *written,
                          int *block_err)
{
    size_t ip = 0, op = 0;
    *written = 0; *block_err = 0;
    while (ip < n) {
        if (n - ip < 4) return LZ4O_FERR_IO_EOF;
        uint32_t magic = ld32(in + ip);
        size_t bs; unsigned flg = 0x20; uint64_t want_size = 0;
        if (magic == F_LEGACY_MAGIC) {
            ip += 4; bs = 8u << 20;
        } else {
            if (n - ip < 7) return LZ4O_FERR_IO_EOF;
            if (magic >= F_SKIP_LO && magic <= F_SKIP_HI) return LZ4O_FERR_SKIPPABLE;
            if (magic != F_MAGIC) return LZ4O_FERR_WRONG_MAGIC;
            size_t h = ip + 4;
            flg = in[h]; uint8_t bd = in[h + 1];
            size_t need = 7 + ((flg & 0x08) ? 8 : 0) + ((flg & 0x01) ? 4 : 0);
            if (n - ip < need) return LZ4O_FERR_IO_EOF;
            if ((flg & 0xC0) != 0x40) return LZ4O_FERR_UNSUPPORTED_VERSION;
            if ((flg & 0x02) || (bd & 0x8F)) return LZ4O_FERR_RESERVED_BITS;
            int id = (bd >> 4) & 7;
            if (id < 4) return LZ4O_FERR_UNSUPPORTED_BLOCKSIZE;
            bs = lz4o_block_size_bytes(id);
            size_t o = h + 2;
            if (flg & 0x08) { memcpy(&want_size, in + o, 8); o += 8; }
            if (flg & 0x01) o += 4;
            if ((uint8_t)(lz4o_xxh32(in + h, o - h, 0) >> 8) != in[o]) return LZ4O_FERR_HEADER_CHECKSUM;
            if (flg & 0x01) return LZ4O_FERR_DICTIONARY;
            ip = o + 1;
        }
        /* BlockMode::Linked (frame/decompress.rs:196-222, 277-305): a block may reference the frame's earlier
         * output.  The reference keeps a prefix + ext_dict window of at least WINDOW_SIZE bytes (all of the
         * frame's output while that is shorter), and offsets are 16-bit, so a block sees exactly
         * "everything this frame has produced so far" as its dictionary. */
        const int linked = !(flg & 0x20);
        const size_t frame_begin = op;
        xxh32_state content; xs_init(&content, 0);
        uint64_t got = 0;
        for (;;) {
            /* frame/decompress.rs:236-243: EOF where a BlockInfo is due ends the read cleanly
             * (this is also how a legacy frame, which has no EndMark, terminates). */
            if (n - ip < 4) { ip = n; break; }
            uint32_t info = ld32(in + ip); ip += 4;
            if (info == 0) {                                          /* EndMark */
                if ((flg & 0x08) && got != want_size) return LZ4O_FERR_CONTENT_LENGTH;
                if (flg & 0x04) {
                    if (n - ip < 4) return LZ4O_FERR_IO_EOF;
                    if (ld32(in + ip) != xs_digest(&content)) return LZ4O_FERR_CONTENT_CHECKSUM;
                    ip += 4;
                }
                break;
            }
            size_t len = info & 0x7FFFFFFFu, produced;
            if (len > bs) return LZ4O_FERR_BLOCK_TOO_BIG;
            if (n - ip < len) return LZ4O_FERR_IO_EOF;
            const uint8_t *payload = in + ip; ip += len;
            if (flg & 0x10) {
                if (n - ip < 4) return LZ4O_FERR_IO_EOF;
                if (ld32(in + ip) != lz4o_xxh32(payload, len, 0)) return LZ4O_FERR_BLOCK_CHECKSUM;
                ip += 4;
            }
            if (info & 0x80000000u) {
                if (cap - op < len) return LZ4O_FERR_OUTPUT_FULL;
                memcpy(out + op, payload, len); produced = len;
            } else {
                size_t room = cap - op < bs ? cap - op : bs, e1, e2;
                int st = linked ? lz4o_decompress_block_dict(payload, len, out + frame_begin, op - frame_begin, out + op,
                                                             room, &produced, &e1, &e2)
                                : lz4o_decompress_block(payload, len, out + op, room, &produced, &e1, &e2);
                if (st != LZ4O_OK) {
                    if (st == LZ4O_ERR_OUTPUT_TOO_SMALL && room < bs) return LZ4O_FERR_OUTPUT_FULL;
                    *block_err = st; return LZ4O_FERR_DECOMPRESSION;
                }
            }
            if (flg & 0x04) xs_update(&content, out + op, produced);
            op += produced; got += produced;
        }
    }
    *written = op;
    return LZ4O_OK;
}

/* ------------------------------------------------------------------------------------------ */
/* batch helpers for the CPU baseline (one block per task, static interleave over threads)     */

#include <pthread.h>

typedef struct {
    int tid, nthreads, decode;
    const uint8_t *in; const uint64_t *in_off; const uint32_t *in_len;
    uint8_t *out; const uint64_t *out_off; const uint32_t *out_cap; uint32_t *out_len; int32_t *status;
    size_t nblocks;
} batch_job;

static void *batch_worker(void *arg)
{
    batch_job *j = (batch_job *)arg;
    uint32_t *tab32 = (uint32_t *)malloc(LZ4O_SLOTS * sizeof(uint32_t));
    for (size_t b = (size_t)j->tid; b < j->nblocks; b += (size_t)j->nthreads) {
        const uint8_t *src = j->in + j->in_off[b];
        uint8_t *dst = j->out + j->out_off[b];
        if (j->decode) {
            size_t w, e1, e2;
            j->status[b] = lz4o_decompress_block(src, j->in_len[b], dst, j->out_cap[b], &w, &e1, &e2);
            j->out_len[b] = (uint32_t)w;
        } else {
            int64_t r;
            if (j->in_len[b] < 65535) {
                r = lz4o_compress_block(src, j->in_len[b], dst, j->out_cap[b]);
            } else {
                memset(tab32, 0, LZ4O_SLOTS * sizeof(uint32_t));
                r = encode_u32_h5(src, j->in_len[b], dst, j->out_cap[b], tab32, 0, NULL, 0);
            }
            j->status[b] = r < 0 ? LZ4O_ERR_COMPRESS_OUTPUT_TOO_SMALL : LZ4O_OK;
            j->out_len[b] = r < 0 ? 0 : (uint32_t)r;
        }
    }
    free(tab32);
    return NULL;
}

static void run_batch(int decode, const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
                      uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
                      uint32_t *out_len, int32_t *status, size_t nblocks, int nthreads)
{
    if (nthreads < 1) nthreads = 1;
    if (nthreads > 256) nthreads = 256;
    pthread_t th[256]; batch_job jobs[256];
    for (int t = 0; t < nthreads; t++) {
        jobs[t] = (batch_job){t, nthreads, decode, in, in_off, in_len, out, out_off, out_cap, out_len, status, nblocks};
        if (t) pthread_create(&th[t], NULL, batch_worker, &jobs[t]);
    }
    batch_worker(&jobs[0]);
    for (int t = 1; t < nthreads; t++) pthread_join(th[t], NULL);
}

void lz4o_compress_batch(const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
                         uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
                         uint32_t *out_len, int32_t *status, size_t nblocks, int nthreads)
{
    run_batch(0, in, in_off, in_len, out, out_off, out_cap, out_len, status, nblocks, nthreads);
}

void lz4o_decompress_batch(const uint8_t *in, const uint64_t *in_off, const uint32_t *in_len,
                           uint8_t *out, const uint64_t *out_off, const uint32_t *out_cap,
                           uint32_t *out_len, int32_t *status, size_t nblocks, int nthreads)
{
    run_batch(1, in, in_off, in_len, out, out_off, out_cap, out_len, status, nblocks, nthreads);
}
