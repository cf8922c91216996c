"""Ad-hoc GPU parity sweep (run on a GPU during development); the real tests are test_gpu_*.py."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import oracle
from lz4_flex_b200 import block, corpus, frame

ctx = block.Context(0)
bad = 0

def check(name, cond):
    global bad
    if not cond:
        bad += 1
        print("FAIL", name)

# fixtures, block API
for f in ["compression_1k.txt", "compression_34k.txt", "compression_65k.txt", "compression_66k_JSON.txt"]:
    d = corpus.load(f)
    c = block.compress(d, ctx=ctx)
    check(f + " compress", c == oracle.compress_block(d))
    check(f + " rt", block.decompress(c, len(d), ctx=ctx) == d)
# edge sizes
rng = np.random.default_rng(1)
cases = [b"", b"a", b"a" * 12, b"a" * 13, b"a" * 14, b"Hello people, what's up?", bytes(30000), bytes(65536),
         bytes(65535), bytes(65534), bytes(65537), rng.integers(0, 256, 65536, dtype=np.uint8).tobytes(),
         rng.integers(0, 4, 100000, dtype=np.uint8).tobytes(), rng.integers(0, 2, 70000, dtype=np.uint8).tobytes()]
for n in [15, 16, 17, 31, 32, 33, 63, 64, 65, 255, 256, 270, 271, 272, 300, 1000, 4096, 65535, 65536, 65537, 70000]:
    cases.append(rng.integers(0, 3, n, dtype=np.uint8).tobytes())
    cases.append((b"abcdefgh" * (n // 8 + 1))[:n])
comp = block.compress_blocks(cases, ctx=ctx)
for i, (d, c) in enumerate(zip(cases, comp)):
    o = oracle.compress_block(d)
    check(f"case {i} len {len(d)} compress ({len(c)} vs {len(o)})", c == o)
outs, status, _ = block.decompress_blocks(comp, [max(len(d), 1) for d in cases], ctx=ctx)
for i, (d, o) in enumerate(zip(cases, outs)):
    check(f"case {i} rt", o == d and status[i] == 0)
# CONT / hash5 modes
fl = [block.BLOCK_CONT | block.BLOCK_HASH5_ALWAYS] * len(cases)
comp = block.compress_blocks(cases, fl, ctx=ctx)
for i, (d, c) in enumerate(zip(cases, comp)):
    check(f"case {i} cont", c == oracle.compress_block_cont(d))
fl = [block.BLOCK_HASH5_ALWAYS] * len(cases)
comp = block.compress_blocks(cases, fl, ctx=ctx)
for i, (d, c) in enumerate(zip(cases, comp)):
    check(f"case {i} fresh-h5", c == oracle.compress_block_fresh_h5(d))
# decode error vectors
vecs = [([0x30, 97, 52, 57], 3), ([], 255), ([0xF0], 255), ([0x0F, 0], 255), ([0x0F, 1, 0], 255), ([0x40, 97, 1, 0], 4),
        ([0x20, 97, 97, 1, 0], 1), ([0x10, 97, 1, 0], 4), ([0x0E, 255] + [0] * 18, 256), ([0x0F, 1, 0, 1, 0x70] + [0] * 20, 256),
        ([0x40, 0, 0, 0, 0, 255, 0, 0x70] + [0] * 20, 256), ([0x0E, 0, 0, 0x70] + [0] * 20, 256), ([0x00], 10)]
outs, status, exp = block.decompress_blocks([bytes(v) for v, _ in vecs], [c for _, c in vecs], ctx=ctx, raise_on_error=False)
for i, (v, cap) in enumerate(vecs):
    st, o, e1, e2 = oracle.decompress_block(bytes(v), cap)
    check(f"vec {i} status {status[i]} vs {st}", status[i] == st and (st != 0 or outs[i] == o) and (st != 2 or exp[i] == e1))
# big: dickens 4 MiB block + tiled json 64 MiB
d = corpus.load("dickens.txt")[: 4 << 20]
t0 = time.time(); c = block.compress(d, ctx=ctx); t1 = time.time()
check("dickens 4MiB compress", c == oracle.compress_block(d))
check("dickens 4MiB rt", block.decompress(c, len(d), ctx=ctx) == d)
data = corpus.tiled("compression_66k_JSON.txt", 64 << 20)
nb = data.size // 65536
offs = np.arange(nb, dtype=np.uint64) * 65536
lens = np.full(nb, 65536, dtype=np.uint32)
t0 = time.time(); out, ooff, olen = block.compress_batch(data, offs, lens, ctx=ctx); t1 = time.time()
print("64MiB json compress host e2e s", t1 - t0, "ratio", olen.sum() / data.size)
dst = np.zeros(int(olen.astype(np.uint64).sum()), dtype=np.uint8)
ool, ost = oracle.compress_batch(data, offs, lens, np.zeros(nb * 72109, dtype=np.uint8), offs * 0 + np.arange(nb, dtype=np.uint64) * 72109, np.full(nb, 72109, dtype=np.uint32), 8)
check("json batch lens", (ool == olen).all())
ob = np.zeros(nb * 72109, dtype=np.uint8)
ool, ost = oracle.compress_batch(data, offs, lens, ob, np.arange(nb, dtype=np.uint64) * 72109, np.full(nb, 72109, dtype=np.uint32), 8)
okb = all(out[int(ooff[b]):int(ooff[b]) + int(olen[b])].tobytes() == ob[b * 72109:b * 72109 + int(ool[b])].tobytes() for b in range(nb))
check("json batch bytes", okb)
back = np.zeros(data.size, dtype=np.uint8)
t0 = time.time(); ol, st, _ = block.decompress_batch(out, ooff, olen, back, offs, lens, ctx=ctx); t1 = time.time()
print("64MiB json decompress host e2e s", t1 - t0)
check("json batch rt", (back == data).all())
# frame
for bsid in (4, 5, 7):
    f = frame.compress_frame(data[: 9 << 20].tobytes(), frame.FrameInfo(block_size=frame.BlockSize(bsid)), ctx=ctx)
    check(f"frame bs{bsid}", f == oracle.frame_compress(data[: 9 << 20].tobytes(), bsid))
    check(f"frame bs{bsid} rt", frame.decompress_frame(f, ctx=ctx) == data[: 9 << 20].tobytes())
f = frame.compress_frame(data[: 3 << 20].tobytes(), frame.FrameInfo(block_size=frame.BlockSize.Max64KB, block_checksums=True, content_checksum=True, content_size=3 << 20), ctx=ctx)
check("frame checksums", f == oracle.frame_compress(data[: 3 << 20].tobytes(), 4, 7))
check("frame checksums rt", frame.decompress_frame(f, ctx=ctx) == data[: 3 << 20].tobytes())
leg = corpus.load("dickens.lz4")
check("legacy frame", frame.decompress_frame(leg, ctx=ctx) == corpus.load("dickens.txt"))
print("FAILURES", bad)
sys.exit(1 if bad else 0)
