"""Development aid (run on a GPU): host-batch call timings for chunk-size / overlap tuning."""
import os, sys, time, threading, queue
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np, torch
from lz4_flex_b200 import block, corpus
nb = 16384; B = 65536
data = corpus.tiled("compression_66k_JSON.txt", nb * B)
h_in = torch.empty(nb * B, dtype=torch.uint8).pin_memory(); h_in.numpy()[:] = data
h_comp = torch.empty(400 << 20, dtype=torch.uint8).pin_memory()
h_back = torch.empty(nb * B, dtype=torch.uint8).pin_memory()
offs = np.arange(nb, dtype=np.uint64) * B; lens = np.full(nb, B, dtype=np.uint32)
ctx = block.Context(0); ctx2 = block.Context(0, high_priority=os.environ.get("PRIO", "1") == "1")
tc, td = [], []
for it in range(4):
    t0 = time.perf_counter(); out, ooff, olen = block.compress_batch(h_in.numpy(), offs, lens, None, out=h_comp.numpy(), ctx=ctx); t1 = time.perf_counter()
    block.decompress_batch(out, ooff, olen, h_back.numpy(), offs, lens, ctx=ctx2); t2 = time.perf_counter()
    if it: tc.append(t1 - t0); td.append(t2 - t1)
assert np.array_equal(h_back.numpy(), data)
print(f"serial: compress call {1e3*np.mean(tc):.2f} ms, decompress call {1e3*np.mean(td):.2f} ms")

def pipelined(nchunks):
    per = -(-nb // nchunks); q = queue.Queue()
    def comp():
        pos = 0; hc = h_comp.numpy()
        for b0 in range(0, nb, per):
            b1 = min(nb, b0 + per)
            o, oo, ol = block.compress_batch(h_in.numpy(), offs[b0:b1], lens[b0:b1], None, out=hc[pos:], ctx=ctx)
            q.put((b0, b1, pos, oo, ol)); pos += int(oo[-1]) + int(ol[-1])
        q.put(None)
    th = threading.Thread(target=comp); th.start(); hc = h_comp.numpy()
    while True:
        it = q.get()
        if it is None: break
        b0, b1, pos, oo, ol = it
        block.decompress_batch(hc[pos:], oo, ol, h_back.numpy(), offs[b0:b1], lens[b0:b1], ctx=ctx2)
    th.join()
for nch in (2, 4, 8):
    ts = []
    for it in range(4):
        h_back.numpy()[::4096] = 0
        torch.cuda.synchronize(); t0 = time.perf_counter(); pipelined(nch); torch.cuda.synchronize(); dt = time.perf_counter() - t0
        if it: ts.append(dt)
    assert np.array_equal(h_back.numpy(), data)
    print(f"pipelined x{nch}: {1e3*np.mean(ts):.2f} ms")
