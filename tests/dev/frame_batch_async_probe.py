"""Development aid: the sync-free batch frame decoder (lz4b200_frame_decompress_batch_device_async) against the
synchronous one (lz4b200_frame_decompress_batch_device, on a context whose frame budget holds every frame in one group).

    python tests/dev/frame_batch_async_probe.py [--out DIR]

Prints the card, its power limit and max SM clock, then for
  (a) 4 096 frames of 256 KiB JSON from compress_frames_device,
  (b) 16 384 single-block frames of 64 KiB JSON,
  (c) 256 linked frames of 1 MiB of dickens in 64 KiB blocks,
  (d) one frame of 256 MiB of hdfs JSON in 64 blocks of 4 MiB,
checks every result and every output byte of the async call against the sync call, then reports (one warm-up, then
three alternating passes, median): the device time of each call (CUDA events around it), how long each call holds
the host before it returns, 20 batches enqueued back to back against 20 synchronous calls (host clock to the end of a
device synchronise), and the replay of the async call captured in a CUDA graph (events).  The async call uses the
default block capacity (default_max_blocks)."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
import oracle  # noqa: E402
from lz4_flex_b200 import _native, block, corpus, frame  # noqa: E402
from stream_frames import linked_frame  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def i64(v):
    return torch.tensor(np.asarray(v, dtype=np.int64), device="cuda")


class Case:
    def __init__(self, name, d_in, offs, lens, raw):
        self.name, self.d_in, self.raw = name, d_in, raw
        self.n = len(offs)
        caps = [len(r) for r in raw]
        oo = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
        self.d_off, self.d_len, self.d_ooff, self.d_cap = i64(offs), i64(lens), i64(oo), i64(caps)
        self.want = torch.from_numpy(np.frombuffer(b"".join(raw), dtype=np.uint8).copy()).cuda()
        self.out_s = torch.empty_like(self.want)
        self.out_a = torch.empty_like(self.want)
        self.res_s = torch.zeros((self.n, 5), dtype=torch.int64, device="cuda")

    def sync(self, ctx):
        st = _native.lib().lz4b200_frame_decompress_batch_device(
            ctx.handle, self.d_in.data_ptr(), self.d_off.data_ptr(), self.d_len.data_ptr(), self.out_s.data_ptr(),
            self.d_ooff.data_ptr(), self.d_cap.data_ptr(), self.res_s.data_ptr(), self.n,
            torch.cuda.current_stream().cuda_stream)
        assert st == 0, ctx.last_cuda_error()

    def run_async(self, ctx):
        return frame.decompress_frames_device_async(self.d_in, self.d_off, self.d_len, self.out_a, self.d_ooff,
                                                    self.d_cap, ctx=ctx).results

    def check(self, res_a):
        torch.cuda.synchronize()
        assert (self.res_s[:, 4] == 0).all() and torch.equal(self.res_s[:, 1].cpu(), self.d_cap.cpu()), self.name
        assert torch.equal(res_a, self.res_s), self.name
        assert torch.equal(self.out_s, self.want) and torch.equal(self.out_a, self.want), self.name


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


def cases(ctx):
    j = corpus.tiled("compression_66k_JSON.txt", 1 << 30)
    d_j = torch.from_numpy(j).cuda()
    out = []
    n = 4096
    offs = np.arange(n, dtype=np.int64) * (256 << 10)
    f, fo = frame.compress_frames_device(d_j, offs, [256 << 10] * n, ctx=ctx)
    fo = fo.cpu().numpy()
    raw = [j[o:o + (256 << 10)].tobytes() for o in offs]
    out.append(Case("4096 x 256 KiB JSON frames", f.clone(), fo[:-1], np.diff(fo), raw))
    n = 16384
    offs = np.arange(n, dtype=np.int64) * 65536
    f, fo = frame.compress_frames_device(d_j, offs, [65536] * n, frame.FrameInfo(block_size=frame.BlockSize.Max64KB),
                                         ctx=ctx)
    fo = fo.cpu().numpy()
    raw = [j[o:o + 65536].tobytes() for o in offs]
    out.append(Case("16384 x 64 KiB JSON single-block frames", f.clone(), fo[:-1], np.diff(fo), raw))
    del d_j, f
    d = corpus.tiled("dickens.txt", 256 << 20)
    raw = [d[i << 20:(i + 1) << 20].tobytes() for i in range(256)]
    fr = [linked_frame(r, [65536], 4, False, True) for r in raw]
    lens = np.array([len(x) for x in fr], dtype=np.int64)
    out.append(Case("256 x 1 MiB linked dickens frames", torch.from_numpy(np.frombuffer(b"".join(fr), np.uint8).copy())
                    .cuda(), np.concatenate([[0], np.cumsum(lens)[:-1]]), lens, raw))
    h = corpus.tiled("hdfs.json", 256 << 20).tobytes()
    fh = oracle.frame_compress(h, 7, oracle.F_CONTENT_CHECKSUM)
    out.append(Case("1 x 64 x 4 MiB hdfs frame", torch.from_numpy(np.frombuffer(fh, np.uint8).copy()).cuda(), [0],
                    [len(fh)], [h]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_batch_async_probe"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    ctx = block.Context(0)
    _native.lib().lz4b200_ctx_set_frame_budget(ctx.handle, 8 << 30)
    report = {"card (name, power limit, max SM clock)": card(), "cases": {}}
    print(report["card (name, power limit, max SM clock)"], flush=True)
    for c in cases(ctx):
        c.sync(ctx)                                                           # warm-up, and the outputs checked
        c.check(c.run_async(ctx))
        g = torch.cuda.CUDAGraph()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            c.run_async(ctx)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        with torch.cuda.graph(g, capture_error_mode="global"):
            gres = c.run_async(ctx)
        c.out_a.zero_()
        g.replay()
        c.check(gres)
        t = {k: [] for k in ("sync device ms", "async device ms", "sync host hold ms", "async host hold ms",
                             "20 sync calls ms", "20 async calls ms", "graph replay device ms")}
        for _ in range(3):                                                    # alternating passes
            t["sync device ms"].append(event_ms(lambda: c.sync(ctx)))
            t["async device ms"].append(event_ms(lambda: c.run_async(ctx)))
            t["sync host hold ms"].append(host_hold_ms(lambda: c.sync(ctx)))
            t["async host hold ms"].append(host_hold_ms(lambda: c.run_async(ctx)))
            t["20 sync calls ms"].append(wall_ms(lambda: c.sync(ctx), 20))
            t["20 async calls ms"].append(wall_ms(lambda: c.run_async(ctx), 20))
            t["graph replay device ms"].append(event_ms(g.replay))
        c.check(c.run_async(ctx))
        row = {k: round(statistics.median(v), 3) for k, v in t.items()}
        row["frames"] = c.n
        row["max_blocks"] = frame.default_max_blocks(c.d_in.numel(), c.n)
        report["cases"][c.name] = row
        print(c.name, json.dumps(row), flush=True)
        del g
    with open(os.path.join(args.out, "frame_batch_async_probe.json"), "w") as fh:
        json.dump(report, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
