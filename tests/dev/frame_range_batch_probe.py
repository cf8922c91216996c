"""Development aid: the batch index (lz4b200_frame_index_batch_device) and the batch range decoder
(lz4b200_frame_decompress_ranges_batch_device) against a host loop of the one-frame calls over the same frames.

    python tests/dev/frame_range_batch_probe.py [--out DIR]

Prints the card and its power limit, checks every output against the source, then for
  (a) 4 096 frames x 256 KiB of JSON in 64 KiB blocks, packed back to back by compress_frames_device;
  (b) 256 linked frames x 1 MiB of dickens in 64 KiB blocks;
times the index build and 10 000 random 4 KiB ranges spread over the frames, batch call against the loop (one warm-up,
then three alternating passes; host clock around calls that end in a device synchronise)."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from lz4_flex_b200 import block, corpus, frame  # noqa: E402
from stream_frames import linked_frame  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) * 1e3


def cases(ctx):
    """(name, frames tensor, frame offsets, frame lengths, content tensor, content offsets, content length per frame)."""
    n, size = 4096, 256 << 10
    src = torch.tensor(corpus.tiled("compression_66k_JSON.txt", n * size), device="cuda")
    starts = np.arange(n, dtype=np.int64) * size
    f, fo = frame.compress_frames_device(src, starts, [size] * n, frame.FrameInfo(block_size=frame.BlockSize.Max64KB),
                                         ctx=ctx)
    fo = fo.cpu().numpy()
    out = [("(a) 4096 x 256 KiB JSON, 64 KiB blocks", f, fo[:-1], np.diff(fo), src, starts, size)]
    d = corpus.load("dickens.txt")
    m, size = 256, 1 << 20
    starts = (np.arange(m, dtype=np.int64) * 33331) % (len(d) - size)
    frames = [linked_frame(d[s:s + size], [65536], 4) for s in starts]
    lens = np.array([len(x) for x in frames], dtype=np.int64)
    offs = np.cumsum(lens) - lens
    f = torch.tensor(np.frombuffer(b"".join(frames), dtype=np.uint8), device="cuda")
    src = torch.tensor(np.frombuffer(d, dtype=np.uint8), device="cuda")
    out.append(("(b) 256 linked x 1 MiB dickens, 64 KiB blocks", f, offs, lens, src, starts, size))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_range_batch_probe"))
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    ctx = block.Context(0)
    rng = np.random.default_rng(1)
    rec = {"card": card(), "cases": []}
    print(rec["card"], flush=True)
    for name, f, offs, lens, src, cstart, size in cases(ctx):
        nf = len(offs)
        ix = frame.index_frames_device(f, offs, lens, ctx)
        assert (ix.content_lens() == size).all(), name
        ones = [frame.index_frame_device(f[int(offs[k]):int(offs[k] + lens[k])], ctx) for k in range(nf)]
        for k in range(0, nf, 97):
            assert bytes(ix.frame(k)._info) == bytes(ones[k]._info) and torch.equal(ix.frame(k).entries, ones[k].entries)
        # 10 000 random 4 KiB ranges over random frames
        nr = 10000
        fr = rng.integers(0, nf, nr)
        st = rng.integers(0, size - 4096, nr)
        ln = np.full(nr, 4096, dtype=np.int64)
        oo = np.arange(nr, dtype=np.int64) * 4096
        out_b = torch.empty(nr * 4096, dtype=torch.uint8, device="cuda")
        out_l = torch.empty(nr * 4096, dtype=torch.uint8, device="cuda")
        d_fr, d_st, d_ln, d_oo = (torch.as_tensor(x, device="cuda") for x in (fr, st, ln, oo))
        frame.decompress_frames_ranges_device(f, ix, d_fr, d_st, d_ln, out=out_b, out_offsets=d_oo, ctx=ctx)
        within = np.tile(np.arange(4096), nr)
        want = src[torch.as_tensor(np.repeat(cstart[fr] + st, 4096) + within, device="cuda")]
        assert torch.equal(out_b, want), name
        per = []                                          # the loop: one call per frame with that frame's ranges
        for k in range(nf):
            sel = np.nonzero(fr == k)[0]
            if sel.size:
                per.append((k, f[int(offs[k]):int(offs[k] + lens[k])], *(torch.as_tensor(x[sel], device="cuda")
                                                                           for x in (st, ln, oo))))

        def loop_ranges():
            for k, region, s_, l_, o_ in per:
                frame.decompress_ranges_device(region, ones[k], s_, l_, out=out_l, out_offsets=o_, ctx=ctx)

        loop_ranges()
        assert torch.equal(out_l, want), name
        calls = {"index batch": lambda: frame.index_frames_device(f, offs, lens, ctx),
                 "index loop": lambda: [frame.index_frame_device(f[int(offs[k]):int(offs[k] + lens[k])], ctx)
                                        for k in range(nf)],
                 "ranges batch": lambda: frame.decompress_frames_ranges_device(f, ix, d_fr, d_st, d_ln, out=out_b,
                                                                               out_offsets=d_oo, ctx=ctx),
                 "ranges loop": loop_ranges}
        for fn in calls.values():
            fn()
        times = {k: [] for k in calls}
        for _ in range(3):
            for k, fn in calls.items():
                times[k].append(timed(fn))
        assert torch.equal(out_b, want) and torch.equal(out_l, want), name
        r = {"case": name, "frames": nf, "blocks": int(ix.entries.shape[0]), "ranges": nr,
             "ms": {k: sorted(round(x, 2) for x in v) for k, v in times.items()},
             "median_ms": {k: round(sorted(v)[1], 2) for k, v in times.items()}}
        rec["cases"].append(r)
        print(json.dumps(r), flush=True)
    with open(os.path.join(a.out, "frame_range_batch_probe.json"), "w") as fh:
        json.dump(rec, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
