"""Development aid (run on a GPU): device-timed kernels for BASELINE configs 3 and 5 (not the bench metric).
config 3: decompress-only, dickens.txt tiled to 1 GiB of 64 KiB blocks (oracle-compressed).
config 5: 64 KiB all-zero blocks and incompressible blocks interleaved, zero fraction sweep."""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np, torch
import oracle
from lz4_flex_b200 import block, corpus

dev = torch.device("cuda", 0); ctx = block.Context(0)
B = 65536; slot = 72112

def timed(fn, reps=5):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps

def run(name, data, nb, decode_only=False):
    offs = np.arange(nb, dtype=np.uint64) * B; lens = np.full(nb, B, dtype=np.uint32)
    soff = np.arange(nb, dtype=np.uint64) * slot; scap = np.full(nb, slot, dtype=np.uint32)
    d_in = torch.from_numpy(data).to(dev)
    d_comp = torch.zeros(nb * slot, dtype=torch.uint8, device=dev); d_back = torch.zeros(nb * B, dtype=torch.uint8, device=dev)
    enc = block.DeviceBatch(offs, lens, soff, scap, None, dev); dec = block.DeviceBatch(soff, lens, offs, lens, None, dev)
    dec.in_len = enc.out_len
    enc.compress(d_in, d_comp, ctx); torch.cuda.synchronize()
    clen = enc.out_len.cpu().numpy().astype(np.uint64)
    # oracle bytes on a sample
    for b in (0, 1, nb // 2, nb - 1):
        got = d_comp[b * slot: b * slot + int(clen[b])].cpu().numpy().tobytes()
        assert got == oracle.compress_block(data[b * B:(b + 1) * B]), (name, b)
    t_c = timed(lambda: enc.compress(d_in, d_comp, ctx))
    t_d = timed(lambda: dec.decompress(d_comp, d_back, ctx))
    assert torch.equal(d_back, d_in), name
    gib = nb * B / 2**30
    print(f"{name}: ratio {clen.sum() / (nb * B):.4f}  compress {t_c:.2f} ms ({gib / t_c * 1e3:.1f} GiB/s)  decompress {t_d:.2f} ms ({gib / t_d * 1e3:.1f} GiB/s)")

nb = 16384
run("config 3 (dickens, 16384 x 64 KiB)", corpus.tiled("dickens.txt", nb * B), nb)
zeros = np.zeros(B, dtype=np.uint8)
rnd = corpus.xorshift64star_bytes(nb * B)
for zf in (0.0, 0.25, 0.5, 0.75, 1.0):
    data = rnd.copy().reshape(nb, B)
    k = int(round(zf * 4))
    for b in range(nb):
        if (b % 4) < k: data[b] = 0
    run(f"config 5 zero fraction {zf:.2f}", data.reshape(-1), nb)
