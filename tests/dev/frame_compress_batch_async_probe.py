"""Development aid: the sync-free batch frame encoder (lz4b200_frame_compress_batch_device_async and its linked form)
against the synchronous one (frame.compress_frames_device / compress_linked_frames_device).

    python tests/dev/frame_compress_batch_async_probe.py [--out DIR]

Prints the card, its power limit and max SM clock, then for
  (a) 16 384 frames of 64 KiB JSON, 64 KiB blocks,
  (b) 4 096 frames of 256 KiB JSON, 256 KiB blocks,
  (c) one frame of 1 GiB JSON, block size Auto (4 MiB blocks),
  (d) 256 linked frames of 1 MiB of dickens in 64 KiB blocks,
checks every output byte and offset of the async call against the sync call, then reports (one warm-up, then three
alternating passes, median): the device time of each call (CUDA events around it), how long each call holds the host
before it returns, 20 calls back to back (host clock to the end of a device synchronise), and the replay of the async
call captured in a CUDA graph (events).  The async call uses the default capacity (default_compress_max_blocks,
max_in_bytes = the input's size) and an out_cap of compress_out_cap()."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from lz4_flex_b200 import block, corpus, frame  # noqa: E402
from lz4_flex_b200.frame import BlockMode, BlockSize, FrameInfo  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


class Case:
    def __init__(self, name, d_in, offs, lens, info: FrameInfo):
        self.name, self.d_in, self.info, self.n = name, d_in, info, len(offs)
        self.offs, self.lens = np.asarray(offs, np.int64), np.asarray(lens, np.int64)
        self.d_off = torch.from_numpy(self.offs).cuda()
        self.d_len = torch.from_numpy(self.lens).cuda()
        self.linked = info.block_mode == BlockMode.Linked
        self.out = torch.empty(frame.compress_out_cap(self.n, d_in.numel(), info), dtype=torch.uint8, device="cuda")

    def sync(self, ctx):
        fn = frame.compress_linked_frames_device if self.linked else frame.compress_frames_device
        return fn(self.d_in, self.offs, self.lens, self.info, ctx=ctx)

    def run_async(self, ctx):
        fn = frame.compress_linked_frames_device_async if self.linked else frame.compress_frames_device_async
        return fn(self.d_in, self.d_off, self.d_len, self.out, frame_info=self.info, ctx=ctx)

    def check(self, want, r):
        torch.cuda.synchronize()
        body, offs = want
        assert torch.equal(r.frame_offsets, offs), self.name
        assert bool((r.statuses == 0).all()), self.name
        assert torch.equal(self.out[:body.numel()], body), self.name


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def host_hold_ms(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    return (t1 - t0) * 1e3


def wall_ms(fn, reps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def cases():
    j = torch.from_numpy(corpus.tiled("compression_66k_JSON.txt", 1 << 30)).cuda()
    yield Case("16384 x 64 KiB JSON", j, np.arange(16384) * 65536, [65536] * 16384,
               FrameInfo(block_size=BlockSize.Max64KB))
    yield Case("4096 x 256 KiB JSON", j, np.arange(4096) * (256 << 10), [256 << 10] * 4096,
               FrameInfo(block_size=BlockSize.Max256KB))
    yield Case("1 x 1 GiB JSON Auto", j, [0], [1 << 30], FrameInfo())
    del j
    d = torch.from_numpy(corpus.tiled("dickens.txt", 256 << 20)).cuda()
    yield Case("256 x 1 MiB dickens linked", d, np.arange(256) << 20, [1 << 20] * 256,
               FrameInfo(block_size=BlockSize.Max64KB, block_mode=BlockMode.Linked))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_compress_batch_async_probe"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    ctx = block.Context(0)
    report = {"card (name, power limit, max SM clock)": card(), "cases": {}}
    print(report["card (name, power limit, max SM clock)"], flush=True)
    for c in cases():
        want = [x.clone() for x in c.sync(ctx)]                               # warm-up, and the outputs checked
        c.check(want, c.run_async(ctx))
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            c.run_async(ctx)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, capture_error_mode="global"):
            gres = c.run_async(ctx)
        c.out.zero_()
        g.replay()
        c.check(want, gres)
        t = {k: [] for k in ("sync device ms", "async device ms", "graph replay device ms", "sync host hold ms",
                             "async host hold ms", "20 sync calls ms", "20 async calls ms")}
        for _ in range(3):                                                    # alternating passes
            t["sync device ms"].append(event_ms(lambda: c.sync(ctx)))
            t["async device ms"].append(event_ms(lambda: c.run_async(ctx)))
            t["graph replay device ms"].append(event_ms(g.replay))
            t["sync host hold ms"].append(host_hold_ms(lambda: c.sync(ctx)))
            t["async host hold ms"].append(host_hold_ms(lambda: c.run_async(ctx)))
            t["20 sync calls ms"].append(wall_ms(lambda: c.sync(ctx), 20))
            t["20 async calls ms"].append(wall_ms(lambda: c.run_async(ctx), 20))
        c.check(want, c.run_async(ctx))
        row = {k: round(statistics.median(v), 3) for k, v in t.items()}
        row["frames"] = c.n
        row["max_blocks"] = frame.default_compress_max_blocks(c.d_in.numel(), c.n)
        report["cases"][c.name] = row
        print(c.name, json.dumps(row), flush=True)
        del g, c, want, gres
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "frame_compress_batch_async_probe.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
