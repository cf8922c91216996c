"""CPU tests of the streaming frame encoder's plan (lz4_flex_b200/csrc/lz4b200_frame_encoder.cuh), compiled for the host
by g++ under AddressSanitizer and UndefinedBehaviorSanitizer (tests/cpp/frame_encoder_host.cpp).  On random sequences of
write lengths, flushes and finishes, over every block size, Auto and several frame budgets, the headers, blocks (length,
stream offset, FRESH/CONT), EndMarks and content-length errors the plan emits, concatenated over the calls, must be what
a Python restatement of FrameEncoder (frame/compress.rs:173-404) emits; every call's groups must be whole groups of the
budget (or the flushed rest), its copies must cover its input, and its bound must be the worst case of what it emits.
Only lengths are simulated.  No GPU needed."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "cpp", "frame_encoder_host.cpp")
HDRS = [os.path.join(os.path.dirname(HERE), "lz4_flex_b200", "csrc", h)
        for h in ("lz4b200_frame_encoder.cuh", "lz4b200_frame_batch.cuh", "lz4b200_frame_walk.cuh")]
API = os.path.join(os.path.dirname(HERE), "include", "lz4b200.h")
EXE = os.path.join(HERE, "cpp", "_build", "frame_encoder_host")

CONT, HASH5_ALWAYS = 1, 2
WRITE, FLUSH, FINISH = 0, 1, 2
CONTENT_LENGTH = 109
WINDOW, LIMIT = 65536, 0x7FFFFFFF
SIZES = {4: 64 << 10, 5: 256 << 10, 6: 1 << 20, 7: 4 << 20}
MiB = 1 << 20


@pytest.fixture(scope="module")
def planner():
    if shutil.which("g++") is None:
        pytest.fail("g++ is required to build the host encoder plan")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(p) for p in [SRC, API] + HDRS):
        tmp = f"{EXE}.tmp{os.getpid()}"
        subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-fno-omit-frame-pointer", "-o", tmp, SRC], check=True)
        os.replace(tmp, EXE)

    def run(blob: bytes):
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
        r = subprocess.run([EXE], input=blob, capture_output=True, env=env)
        assert r.returncode == 0 and not r.stderr, r.stderr.decode(errors="replace")[-4000:]
        return [tuple(map(int, ln.split())) for ln in r.stdout.decode().splitlines()]
    return run


def auto_id(n):
    return 7 if n > 256 << 10 else 5 if n > 64 << 10 else 4


def slot(n):
    return (20 + n * 110 // 100 + 15) & ~15                 # lz4b200_max_output_size(n), rounded up to 16


def group_blocks(bs, budget):
    return max(1, budget // (bs + slot(bs)))


class RefEncoder:
    """FrameEncoder (compress.rs:173-404) over lengths: the events it writes, in order."""

    def __init__(self, bsid, content_size):
        self.bsid, self.content_size = bsid, content_size
        self.open = self.written = False
        self.src = self.so = self.cl = 0
        self.ev = []

    def begin(self, n):                                     # compress.rs:234-258
        self.open = True
        if self.bsid == 0:
            self.bsid = auto_id(n)
        self.ev.append(("H",))
        if self.cl:
            self.cl = self.so = self.src = 0

    def write_block(self):                                  # compress.rs:261-371
        bs = SIZES[self.bsid]
        if self.so + bs + WINDOW >= LIMIT:
            self.so = 0
        self.ev.append(("B", self.src, self.so, HASH5_ALWAYS | (CONT if self.so else 0)))
        self.cl += self.src
        self.so += self.src
        self.src = 0

    def write(self, n):                                     # compress.rs:375-396
        if not self.open and n:
            self.begin(n)
        while n:
            room = SIZES[self.bsid] - self.src
            if room == 0:
                self.write_block()
                continue
            t = min(room, n)
            self.src += t
            n -= t

    def flush(self):
        if self.src:
            self.write_block()

    def finish(self):                                       # compress.rs:173-187, 209-230
        self.flush()
        if not self.open and not self.written:
            self.begin(0)
        self.open = False
        if self.content_size is not None and self.content_size != self.cl:
            self.ev.append(("X", self.content_size, self.cl))
            return CONTENT_LENGTH
        self.ev.append(("E",))
        self.written = True
        return 0


def record(bsid, bc, cc, content_size, budget, ops):
    head = struct.pack("<IiBBBQQ", len(ops), bsid, bc, cc, content_size is not None, content_size or 0, budget)
    return head + b"".join(struct.pack("<QB", n, op) for n, op in ops)


def check_case(out, pos, case):
    """Checks one sequence's calls from out[pos:]; returns the position after them."""
    bsid, bc, cc, content_size, budget, ops = case
    ref = RefEncoder(bsid, content_size)
    hdr_len = 15 if content_size is not None else 7
    got_ev, buffered, group = [], 0, 0
    for n, op in ops:
        ref.write(n)
        want_status = 0
        if op == FLUSH:
            ref.flush()
        elif op == FINISH:
            want_status = ref.finish()
        status, header, endmark, rid, g, bound, nsteps, nblocks, buf_after, cl_after = out[pos]
        steps = out[pos + 1:pos + 1 + nsteps]
        blocks = out[pos + 1 + nsteps:pos + 1 + nsteps + nblocks]
        pos += 1 + nsteps + nblocks
        assert status == want_status
        assert rid == ref.bsid
        if rid == 0:                                        # Auto, and no frame has opened yet: nothing happens
            assert (header, endmark, nsteps, nblocks, bound) == (0, 0, 0, 0, 0)
            continue
        bs = SIZES[rid]
        if header:
            got_ev.append(("H",))
            group = g
            assert g == group_blocks(bs, budget)
            buffered = 0
        assert g == group or not group
        # the copies cover the call's input in order, into the buffer after what it holds
        src = 0
        emitted = hdr_len * header
        for s_src, s_dst, s_len, s_glen, s_nb, s_f0 in steps:
            assert s_src == src and (s_len == 0 or s_dst == buffered)
            src += s_len
            buffered += s_len
            if s_glen:
                assert s_glen == buffered and s_nb == -(-s_glen // bs)
                assert s_glen == g * bs or (op != WRITE and src == n and s_glen < g * bs)
                for k in range(s_nb):
                    ln = min(bs, s_glen - k * bs)
                    fl, off = blocks[s_f0 + k]
                    got_ev.append(("B", ln, off, fl))
                    emitted += 4 + ln + 4 * bc
                buffered = 0
            assert buffered < g * bs
        assert src == n and buffered == buf_after
        if op == FINISH:
            emitted += 8 if cc else 4
        if endmark:
            got_ev.append(("E",))
        if status == CONTENT_LENGTH:
            got_ev.append(("X", content_size, cl_after))
        assert bound == emitted
        if op != WRITE:                                     # both have written every block
            assert got_ev == ref.ev
    # after a WRITE, the plan may still buffer blocks the reference has written, and may have compressed the full block
    # the reference keeps until more input or a flush comes
    if len(got_ev) > len(ref.ev):
        assert ref.src == SIZES[ref.bsid]
        ref.write_block()
    assert got_ev == ref.ev[:len(got_ev)]
    assert all(e[0] == "B" for e in ref.ev[len(got_ev):])
    return pos


def random_ops(rng, bs_hint):
    ops = []
    for _ in range(int(rng.integers(1, 14))):
        r = rng.random()
        bs = bs_hint
        if r < 0.12:
            n = 0
        elif r < 0.24:
            n = 1
        elif r < 0.5:
            n = int(rng.choice([bs - 1, bs, bs + 1, 2 * bs, 3 * bs - 1]))
        elif r < 0.8:
            n = int(rng.integers(0, 3 * bs))
        else:
            n = int(rng.integers(1, 40)) * bs + int(rng.integers(-1, 2))
        n = max(n, 0)
        q = rng.random()
        op = WRITE if q < 0.55 else FLUSH if q < 0.8 else FINISH
        ops.append((n, op))
    return ops


def random_case(rng):
    bsid = int(rng.choice([0, 4, 5, 6, 7]))
    budget = int(rng.choice([MiB, 3 * MiB, 16 * MiB, 256 * MiB, 2048 * MiB]))
    hint = SIZES[bsid] if bsid else int(rng.choice([64 << 10, 256 << 10, 4 << 20]))
    if bsid == 0 and rng.random() < 0.5:
        hint = 65536
    ops = random_ops(rng, hint)
    content_size = None
    if rng.random() < 0.3:
        content_size = int(rng.choice([0, 1, sum(n for n, _ in ops), sum(n for n, _ in ops[:2])]))
    return bsid, int(rng.integers(0, 2)), int(rng.integers(0, 2)), content_size, budget, ops


def reposition_case(rng):
    """A frame that crosses the 2 GiB reposition after an early flush shifted the phase."""
    bsid = int(rng.choice([4, 7, 0]))
    bs = SIZES[bsid] if bsid else 4 << 20
    first = int(rng.integers(1, bs))                       # a short block: every later offset is off the block grid
    big = (LIMIT // bs + int(rng.integers(-3, 4))) * bs
    ops = [(first if bsid else bs + 1, FLUSH), (big, WRITE), (int(rng.integers(0, 5 * bs)), int(rng.choice([1, 2]))),
           (int(rng.integers(0, 3)) * bs, FINISH), (bs + 7, WRITE), (bs, FINISH)]
    return bsid, 0, 1, None, int(rng.choice([MiB, 256 * MiB])), ops


def test_plan_matches_restatement(planner):
    rng = np.random.default_rng(11)
    cases = [random_case(rng) for _ in range(3000)] + [reposition_case(rng) for _ in range(12)]
    out = planner(b"".join(record(*c) for c in cases))
    pos = 0
    for c in cases:
        pos = check_case(out, pos, c)
    assert pos == len(out)


def test_reposition_after_flush_is_not_the_block_index(planner):
    """After a 1-byte flush, the first block that reaches the reposition is FRESH at its stream offset, which is not
    where k % fresh_period puts it; every block after a reposition restarts from offset 0."""
    bs = 64 << 10
    ops = [(1, FLUSH), (LIMIT // bs * bs, WRITE), (bs, FINISH)]
    case = (4, 0, 0, None, 256 * MiB, ops)
    out = planner(record(*case))
    assert check_case(out, 0, case) == len(out)
    ref = RefEncoder(4, None)
    ref.write(1); ref.flush(); ref.write(ops[1][0]); ref.write(bs); ref.finish()
    fresh = [k for k, e in enumerate(x for x in ref.ev if x[0] == "B") if not e[3] & CONT]
    period = -(-(LIMIT - WINDOW - bs) // bs)
    assert fresh[0] == 0 and len(fresh) == 2 and fresh[1] != period


def test_quirks(planner):
    """Empty finish: an empty frame; second finish: a second EndMark; Auto resolves once; state resets only after
    content; a content-length error closes the frame without an EndMark."""
    cases = [
        (0, 0, 1, None, 256 * MiB, [(0, FINISH), (0, FINISH), (300 << 10, WRITE), (0, FINISH), (5, FINISH)]),
        (0, 1, 0, 10, 16 * MiB, [(0, FINISH), (10, WRITE), (0, FINISH), (0, FINISH), (11, FINISH), (10, FINISH)]),
        (5, 0, 0, None, MiB, [(0, WRITE), (0, FLUSH), (1, WRITE), (0, FLUSH), (0, FLUSH), (9 << 20, FINISH)]),
    ]
    out = planner(b"".join(record(*c) for c in cases))
    pos = 0
    for c in cases:
        pos = check_case(out, pos, c)
    assert pos == len(out)
    # the first: Auto took 64 KiB from the empty finish, and kept it for the 300 KiB write
    assert out[0][3] == 4 and out[2][3] == 4


def test_group_of_the_default_budget():
    assert group_blocks(64 << 10, 256 * MiB) == 1950
    assert 65536 + slot(65536) == 65536 + 72112
    assert group_blocks(4 << 20, 16 * MiB) == 1 and group_blocks(4 << 20, MiB) == 1
