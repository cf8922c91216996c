"""CPU model of a window walk for K2 (DESIGN.md §6, "Window walk": built, measured slower than the one-sequence walk,
not kept).  A group of G lanes reads W = G * B compressed bytes as aligned words (never a word that holds no byte of the
stream), every lane sizes the sequence that would start at each of its B byte positions, the chain from the cursor picks
up to G of them, a scan places them in the output, and the fast path's checks cut the window at the first sequence that
fails one; that sequence goes through the one-sequence step.  Copies: literals and the short matches whose source ends
before the window's first output byte are all loaded before any store of the window; the other matches follow in
stream order.

The model keeps the lane arithmetic of the measured kernel with G and B as parameters and is checked against the serial
walk (one sequence at a time, reference src/block/decompress.rs:330-444): same sequence boundaries, same window-ending
sequence, same output bytes, same status and `expected`.  It also reports how many sequences a window holds and how many
matches wait for stream order on the bench's blocks, the figures DESIGN.md §6 quotes as model estimates."""
from __future__ import annotations

import pytest

import oracle
from lz4_flex_b200 import corpus
from test_gpu_launch_shapes import decode_blocks

OK, TOO_SMALL, LIT_OOB, ANOTHER, OFF0, OFF_OOB = 0, 2, 3, 4, 5, 6
SHORT_MATCH = 32                 # longest match a lane copies by itself


class Fail(Exception):
    def __init__(self, status, expected=0):
        self.status, self.expected = status, expected


def fast_seq(src, ip, op, cap):
    """The old fast path's reading of the sequence at ip: (lit, dist, mlen, next ip), or None when it does not apply."""
    n = len(src)
    if ip + 8 > n:
        return None
    tok = src[ip]
    lit = tok >> 4
    q = ip + 1 + lit
    if lit == 15 or q + 8 > n:
        return None
    dist = src[q] | (src[q + 1] << 8)
    mlen, adv = 4 + (tok & 15), 2
    if mlen == 19:
        mlen += src[q + 2]
        adv = 3
    if mlen == 19 + 255 or lit + mlen > cap - op:
        return None
    return lit, dist, mlen, q + adv


def serial_step(src, ip, out, cap):
    """One sequence, every check in the reference's order (decode_block_simple / decode_sequence_checked).  Appends to `out`;
    returns the next ip, or None when the stream ended cleanly."""
    n, op = len(src), len(out)
    f = fast_seq(src, ip, op, cap)
    if f is not None:
        lit, dist, mlen, nxt = f
        out += src[ip + 1: ip + 1 + lit]
        if dist == 0:
            raise Fail(OFF0)
        if dist > len(out):
            raise Fail(OFF_OOB)
        for _ in range(mlen):
            out.append(out[-dist])
        return nxt
    tok = src[ip]
    ip += 1
    lit = tok >> 4
    if lit == 15:
        while True:
            if ip >= n:
                raise Fail(ANOTHER)
            b = src[ip]
            ip += 1
            lit += b
            if b != 255:
                break
    if lit:
        if lit > n - ip:
            raise Fail(LIT_OOB)
        if lit > cap - op:
            raise Fail(TOO_SMALL, op + lit)
        out += src[ip: ip + lit]
        ip += lit
        op += lit
    if ip >= n:
        return None
    if n - ip < 2:
        raise Fail(ANOTHER)
    dist = src[ip] | (src[ip + 1] << 8)
    ip += 2
    if dist == 0:
        raise Fail(OFF0)
    mlen = 4 + (tok & 15)
    if mlen == 19:
        while True:
            if ip >= n:
                raise Fail(ANOTHER)
            b = src[ip]
            ip += 1
            mlen += b
            if b != 255:
                break
    if dist > op:
        raise Fail(OFF_OOB)
    if mlen > cap - op:
        raise Fail(TOO_SMALL, op + mlen)
    for _ in range(mlen):
        out.append(out[-dist])
    if ip >= n:
        raise Fail(ANOTHER)
    return ip


def serial_walk(src, cap):
    """(status, output, expected, token positions) of the one-sequence-at-a-time walk."""
    out, ip, starts = bytearray(), 0, []
    if not src:
        return ANOTHER, b"", 0, starts
    try:
        while ip is not None:
            starts.append(ip)
            ip = serial_step(src, ip, out, cap)
    except Fail as e:
        return e.status, bytes(out), e.expected, starts
    return OK, bytes(out), 0, starts


def window_walk(src, cap, G, B, mis=0, stats=None):
    """The measured kernel's window walk, lane by lane.  `mis` = the stream's address modulo 4."""
    n, W, nwords = len(src), G * B, (mis + len(src) + 3) >> 2
    junk = bytes((i * 37 + 11) & 255 for i in range(4 * (W // 4 + 2)))
    mem = junk[:mis] + bytes(src) + junk                               # whatever the words around the stream hold
    out, ip, starts = bytearray(), 0, []
    if n == 0:
        return ANOTHER, b"", 0, starts
    try:
        while True:
            # (a) aligned words from the one holding ip; words past the stream are not read (0 in the kernel)
            x0 = ip + mis
            wp = ip - (x0 & 3)
            win = bytearray()
            for idx in range((x0 >> 2), (x0 >> 2) + W // 4):
                win += mem[4 * idx: 4 * idx + 4] if idx < nwords else bytes(4)
            win += junk[:32]                                           # the next group's window, or padding
            # (b) every lane sizes every candidate of its B bytes
            nxt = [None] * W
            for lane in range(G):
                for c in range(B):
                    j = lane * B + c
                    tok = win[j]
                    lit, q = tok >> 4, j + 1 + (tok >> 4)
                    mlen, adv = 4 + (tok & 15), 2
                    if mlen == 19:
                        mlen, adv = mlen + win[q + 2], 3
                    ok = lit != 15 and q + adv <= W and mlen != 19 + 255 and wp + j + 8 <= n and wp + q + 8 <= n
                    nxt[j] = q + adv if ok else None
            # (c) the chain from ip, at most G sequences; each lane re-reads its own
            cur, chain = ip - wp, []
            while len(chain) < G and cur < W and nxt[cur] is not None:
                chain.append(cur)
                cur = nxt[cur]
            seqs = []
            for j in chain:
                tok = win[j]
                lit, q = tok >> 4, j + 1 + (tok >> 4)
                mlen = 4 + (tok & 15) + (win[q + 2] if (tok & 15) == 15 else 0)
                seqs.append((j, lit, win[q] | (win[q + 1] << 8), mlen, nxt[j]))
            op0, start, kk = len(out), len(out), len(seqs)
            for s, (j, lit, dist, mlen, _) in enumerate(seqs):          # scan + the fast path's checks
                if not (lit + mlen <= cap - start and dist != 0 and dist <= start + lit):
                    kk = s
                    break
                start += lit + mlen
            if kk == 0:
                starts.append(ip)
                ip = serial_step(src, ip, out, cap)
                if ip is None:
                    break
                continue
            # the window ends where the serial walk leaves the fast path or the window, or after G sequences
            if kk < len(seqs):                                         # cut by a check: the serial walk's too
                f = fast_seq(src, wp + seqs[kk][0], start, cap)
                assert f is None or f[1] == 0 or f[1] > start + f[0], (ip, kk)
            elif kk < G and cur < W:                                   # cut by sizing
                f = fast_seq(src, wp + cur, start, cap)
                assert f is None or f[3] - wp > W, (ip, kk)
            # (d) loads first: literals and the independent short matches read the state before the window
            snap = bytes(out)
            pos, later = op0, []
            buf = bytearray(out) + bytearray(sum(l + m for _, l, _, m, _ in seqs[:kk]))
            for j, lit, dist, mlen, _ in seqs[:kk]:
                starts.append(wp + j)
                buf[pos: pos + lit] = win[j + 1: j + 1 + lit]
                at = pos + lit
                if at - dist + mlen <= op0 and mlen <= SHORT_MATCH:
                    buf[at: at + mlen] = snap[at - dist: at - dist + mlen]
                else:
                    later.append((at, dist, mlen))
                pos = at + mlen
            for at, dist, mlen in later:                                # stream order, byte-serial (copy_match)
                for i in range(mlen):
                    buf[at + i] = buf[at - dist + i]
            out[:] = buf
            if stats is not None:
                stats["windows"] += 1
                stats["seqs"] += kk
                stats["later"] += len(later)
            ip = wp + seqs[kk - 1][4]
    except Fail as e:
        return e.status, bytes(out), e.expected, starts
    return OK, bytes(out), 0, starts


def check(src, cap, G, B, mis=0):
    want = serial_walk(src, cap)
    got = window_walk(src, cap, G, B, mis)
    assert got[0] == want[0] and got[2] == want[2], (got[0], want[0], got[2], want[2])
    assert got[3] == want[3]
    if want[0] == OK:
        assert got[1] == want[1]
    return want


def _blocks(name, count, size=65536):
    t = corpus.tiled(name, count * size)
    return [t[i * size:(i + 1) * size].tobytes() for i in range(count)]


@pytest.mark.parametrize("G,B", [(8, 4), (8, 8), (16, 4), (32, 4), (4, 4)])
@pytest.mark.parametrize("name", ["compression_66k_JSON.txt", "dickens.txt", "hdfs.json"])
def test_window_walk_equals_serial_walk_on_oracle_blocks(name, G, B):
    for i, data in enumerate(_blocks(name, 2, 16384)):
        comp = oracle.compress_block(data)
        st, out, _, _ = check(comp, len(data), G, B, mis=i % 4)
        assert st == OK and out == data


@pytest.mark.parametrize("G,B", [(8, 4), (8, 8), (32, 4)])
def test_window_walk_equals_serial_walk_on_adversarial_vectors(G, B):
    for i, (kind, s, cap, _) in enumerate(decode_blocks(600)):
        st, out, exp, _ = check(s, cap, G, B, mis=i % 4)
        ost, oout, oexp, _ = oracle.decompress_block(s, cap)
        assert st == ost, kind
        if st == OK:
            assert out == oout, kind
        elif st == TOO_SMALL:
            assert exp == oexp, kind


@pytest.mark.parametrize("B", [4, 8])
def test_window_model_figures_on_bench_blocks(B):
    """Sequences per window and matches left for stream order, G = 8, on 64 KiB JSON blocks as the bench builds them."""
    stats = {"windows": 0, "seqs": 0, "later": 0}
    for data in _blocks("compression_66k_JSON.txt", 2):
        comp = oracle.compress_block(data)
        st, out, _, _ = window_walk(comp, len(data), 8, B, stats=stats)
        assert st == OK and out == data
    per_window = stats["seqs"] / stats["windows"]
    print(f"B={B}: {per_window:.2f} sequences per window, {stats['later'] / stats['seqs']:.3f} of matches in stream order")
    assert 1 <= per_window <= 8
