"""CPU model of the block encoder's probe batch with its candidate loads in two tiers (lz4b200_enc_split.cuh,
match_block_view with a WordView), and the seeded blocks that the tier tests run through it and through the GPU.

A batch evaluates the next 32 probe positions of compress.rs:373-439 at once, one per lane, against the table's pre-batch
candidates.  The kernel loads lanes 0..T-1's candidates (tier 1) and the other lanes' (tier 2) as separate loads and
decides from tier 1 alone when tier 1 has a hit w0 and no probe up to w0 shares its slot with an earlier probe of the
batch.  Otherwise it reads tier 2 and resolves the batch exactly as the one-tier matcher does.  The model keeps tier 2's
results unknown until that point, so an output equal to the oracle's shows that tier 1's decisions never needed them.
"""
import numpy as np

from lz4_flex_b200 import corpus

INVALID = 0xFFFFFFFF
MASK64 = (1 << 64) - 1
G = 32


def _h4(b, p):
    v = int.from_bytes(b[p:p + 4], "little")
    return ((v * 2654435761) & 0xFFFFFFFF) >> 20


def _h5(b, p):
    v = int.from_bytes(b[p:p + 8], "little")                     # the reference reads 8 bytes, hashes the low 5
    return ((((v << 24) & MASK64) * 889523592379) & MASK64) >> 52


def _ext(v):
    out = bytearray()
    while v >= 255:
        out.append(255); v -= 255
    out.append(v)
    return bytes(out)


def _last_literals(b, start):
    n = len(b) - start
    return bytes([min(n, 15) << 4]) + (_ext(n - 15) if n >= 15 else b"") + b[start:]


EVENTS = ("batches", "tier1_decided", "tier2_read", "straddle", "invalidated", "end_in_tier2")


def tiered_encode(b: bytes, T: int, cont: bool = False, h5=None, stats=None) -> bytes:
    """One block through the tiered matcher.  `stats` (a dict) counts per batch:
    first_hit[w]  the batch's first real hit is lane w (after forwarding; 32 = none);
    tier1_decided / tier2_read  whether tier 2's candidates were read;
    straddle      two probes up to the winner share a slot, one in each tier;
    invalidated   tier 1's speculative hit was taken away by a slot collision;
    end_in_tier2  the block's last probe position ends the parse inside tier 2."""
    assert 1 <= T < G
    n = len(b)
    if n < 13:
        return _last_literals(b, 0)
    if h5 is None:
        h5 = n >= 65535
    H = _h5 if h5 else _h4
    st = stats if stats is not None else {}
    for e in EVENTS:
        st.setdefault(e, 0)
    first_hit = st.setdefault("first_hit", [0] * (G + 1))
    tab = [INVALID if cont else 0] * 4096
    last_probe, lim = n - 12, n - 6
    out = bytearray()
    anchor = cur = 0
    ri = False
    if not cont:
        tab[H(b, 0)] = 0
        cur = 1
    R = range(G)
    while True:
        base, stride = cur, 1
        while True:
            st["batches"] += 1
            p = [base + i * stride for i in R]
            term = [x > last_probe for x in p]
            if ri:                                               # re-insert of the previous sequence
                tab[H(b, cur - 2)] = cur - 2
                ri = False
            key = [H(b, p[i]) if not term[i] else (0x10000 | i) for i in R]
            cnd = [tab[key[i]] if not term[i] else INVALID for i in R]

            def check(i, c):
                if term[i] or c == INVALID or p[i] - c > 65535:
                    return False
                return b[c:c + 4] == b[p[i]:p[i] + 4]

            hit = [check(i, cnd[i]) if i < T else None for i in R]      # None: tier 2, not read yet
            t1 = [i for i in range(T) if hit[i]]
            w0 = t1[0] if t1 else G
            exact = w0 == 0
            if 1 <= w0 <= 3:                                     # three shuffles: keys of lanes 0..2 against lanes <= w0
                exact = not any(key[j] == key[i] for j in range(1, w0 + 1) for i in range(j))
            same = [[i] for i in R]
            if exact:
                st["tier1_decided"] += 1
                full = [check(i, cnd[i]) for i in R]             # what the one-tier matcher would have seen
                assert full.index(True) == w0
            else:
                st["tier2_read"] += 1
                for i in range(T, G):
                    hit[i] = check(i, cnd[i])
                w0 = hit.index(True) if True in hit else G
                same = [[j for j in R if key[j] == key[i]] for i in R]
                prior = [[j for j in same[i] if j < i] for i in R]
                upto0 = G - 1 if w0 >= G - 1 else w0
                if any(prior[i] for i in range(upto0 + 1)):
                    for i in R:
                        if prior[i]:
                            cnd[i] = p[prior[i][-1]]
                            hit[i] = check(i, cnd[i])
            assert None not in hit[:(hit.index(True) if True in hit else G)]
            win = hit.index(True) if True in hit else G
            tfirst = term.index(True) if True in term else G
            if not exact and w0 < T and win != w0:
                st["invalidated"] += 1
            span = min(win, tfirst)
            if any(key[j] == key[i] for j in range(T, min(span, G - 1) + 1) for i in range(T) if i < j):
                st["straddle"] += 1
            if tfirst < win:                                     # compress.rs:381-384
                first_hit[G] += 1
                if T <= tfirst < G:
                    st["end_in_tier2"] += 1
                return bytes(out) + _last_literals(b, anchor)
            first_hit[win] += 1
            upto = win if win < G else G - 1
            for i in range(upto + 1):                            # commit: last writer per slot among the executed probes
                if max(j for j in same[i] if j <= upto) == i:
                    tab[key[i]] = p[i]
            if win < G:
                mpos, cand = p[win], cnd[win]
                break
            base += G * stride
            stride += 1
        dist = mpos - cand
        while cand > 0 and mpos > anchor and b[mpos - 1] == b[cand - 1]:
            mpos -= 1; cand -= 1
        end, c = mpos + 4, cand + 4
        while end < lim and b[end] == b[c]:
            end += 1; c += 1
        lit, extra = mpos - anchor, end - mpos - 4
        out.append((min(lit, 15) << 4) | min(extra, 15))
        if lit >= 15:
            out += _ext(lit - 15)
        out += b[anchor:mpos]
        out += dist.to_bytes(2, "little")
        if extra >= 15:
            out += _ext(extra - 15)
        anchor = cur = end
        ri = True


# ---- blocks aimed at the tier boundary ------------------------------------------------------------------------------

def _gapped(rng, src: bytes, n: int, gaps) -> bytes:
    """Copies of 12..24 bytes of `src` (text, so the copies' starts were probed and sit in the table) separated by gaps
    of fresh random bytes: after each match the next probe batch's first hit lands about `gap` lanes in."""
    out = bytearray(src[:2048])
    i = 0
    while len(out) < n:
        g = int(gaps[i % len(gaps)]); i += 1
        out += rng.integers(0, 256, g, dtype=np.uint8).tobytes()
        o = int(rng.integers(0, min(len(src), len(out)) - 32))
        out += src[o:o + int(rng.integers(12, 25))]
    return bytes(out[:n])


def _periodic(rng, n: int, period: int) -> bytes:
    """A low-entropy stream whose 4-byte windows repeat every `period` bytes, with sparse flips: probes `period` lanes
    apart share a slot, so collisions cross the tier boundary at every T <= period."""
    unit = rng.integers(0, 4, period, dtype=np.uint8)
    a = np.resize(unit, n)
    flips = rng.random(n) < 0.03
    a[flips] = rng.integers(0, 4, int(flips.sum()), dtype=np.uint8)
    return a.tobytes()


def boundary_blocks(seed: int = 5):
    """(name, data) blocks, seeded: planted first hits at every lane around T = 2, 4 and 8, slot collisions that straddle
    those boundaries (with and without a tier-1 hit they invalidate), and short blocks whose last probe ends the parse in
    any lane."""
    rng = np.random.default_rng(seed)
    json = corpus.load("compression_66k_JSON.txt")
    text = corpus.load("compression_65k.txt")
    out = []
    for T in (2, 4, 8):
        for k in (T - 1, T, T + 1):
            out.append((f"gap{k}_json", _gapped(rng, json, 16384, [k])))
            out.append((f"gap{k}_text", _gapped(rng, text, 16384, [k, k, k + 2])))
    out.append(("gap_mixed", _gapped(rng, json, 65536, rng.integers(0, 12, 64))))
    for period in (3, 5, 6, 9, 12):
        out.append((f"period{period}", _periodic(rng, 12000, period)))
    for k in range(6):
        out.append((f"low_entropy_{k}", rng.integers(0, 2 + k % 3, int(rng.integers(2000, 9000)), dtype=np.uint8).tobytes()))
    for n in list(range(13, 80)) + [95, 140, 300]:               # the last batch's term lanes start at every lane
        out.append((f"tail_random_{n}", rng.integers(0, 256, n, dtype=np.uint8).tobytes()))
        o = int(rng.integers(0, len(json) - n))
        out.append((f"tail_json_{n}", json[o:o + n]))
    return out
