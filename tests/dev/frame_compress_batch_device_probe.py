"""Development aid: the batch frame encoder (lz4b200_frame_compress_batch_device) against the block-batch floor
(lz4b200_compress_batch_device on the same blocks), the one-frame device call (lz4b200_frame_compress_device) in a loop,
and the one-frame call on the whole input as a single frame.

    python tests/dev/frame_compress_batch_device_probe.py [--out DIR]

Prints the card and its power limit, checks every batch output against the C oracle, then for
  (a) 16 384 frames of 64 KiB JSON (1 GiB), no checksums: the batch call, the floor, and the one-frame loop over the
      first 512 frames (reported per frame);
  (b) the same frames with block and content checksums: the batch call and the one-frame loop;
  (c) 262 144 frames of 4 KiB JSON (1 GiB), no checksums: the batch call and the floor;
  (d) 256 frames of 4 MiB hdfs with block checksums: the batch call, and the one-frame call on the same 1 GiB as one
      frame
times each call (one warm-up, then two alternating passes; host clock around calls that end in a device synchronise),
and the host time until the batch call returns (its planning and the upload of the plan, after a synchronise).
A separate profiled batch call per case gives the device time of each kernel (torch.profiler)."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import oracle  # noqa: E402
from frame_batch_device_probe import card, kernel_times, timed  # noqa: E402
from lz4_flex_b200 import _native, block, corpus  # noqa: E402
from lz4_flex_b200.frame import BlockSize, FrameInfo  # noqa: E402

GIB = 1 << 30
HASH5_ALWAYS = 2


class Case:
    def __init__(self, data: np.ndarray, frame_len: int, info: FrameInfo, flags: int):
        self.n = data.size // frame_len
        self.frame_len, self.info, self.flags = frame_len, info, flags
        self.data = data
        self.d_in = torch.from_numpy(data).cuda()
        self.off = np.arange(self.n, dtype=np.int64) * frame_len
        self.len = np.full(self.n, frame_len, dtype=np.int64)
        ci = info.to_c()
        self.cap = self.n * _native.lib().lz4b200_frame_bound(frame_len, C.byref(ci))
        self.d_out = torch.empty(self.cap, dtype=torch.uint8, device="cuda")
        self.d_foff = torch.empty(self.n + 1, dtype=torch.int64, device="cuda")

    def batch(self, ctx):
        ci = self.info.to_c()
        st = _native.lib().lz4b200_frame_compress_batch_device(
            ctx.handle, self.d_in.data_ptr(), self.off.ctypes.data, self.len.ctypes.data, C.byref(ci),
            self.d_out.data_ptr(), self.cap, self.d_foff.data_ptr(), self.n, torch.cuda.current_stream().cuda_stream)
        assert st == 0, ctx.last_cuda_error()

    def loop(self, ctx, count):
        """The one-frame device call on each of the first `count` frames, into the same output places."""
        ci = self.info.to_c()
        s = torch.cuda.current_stream().cuda_stream
        one = self.cap // self.n
        for i in range(count):
            st = _native.lib().lz4b200_frame_compress_device(
                ctx.handle, self.d_in.data_ptr() + int(self.off[i]), self.frame_len, C.byref(ci), self.frame_len,
                self.d_out.data_ptr() + i * one, one, self.d_foff[i:].data_ptr(), s)
            assert st == 0, st

    def floor(self, ctx):
        """The same blocks through lz4b200_compress_batch_device (every block FRESH, as block 0 of its frame)."""
        bs = min(self.frame_len, self.info.block_size.get_size())
        nb = self.data.size // bs
        if not hasattr(self, "_f"):
            slot = (_native.lib().lz4b200_max_output_size(bs) + 15) & ~15
            self._f = dict(off=torch.arange(nb, dtype=torch.int64, device="cuda") * bs,
                           len=torch.full((nb,), bs, dtype=torch.int32, device="cuda"),
                           flags=torch.full((nb,), HASH5_ALWAYS, dtype=torch.uint8, device="cuda"),
                           out=torch.empty(nb * slot, dtype=torch.uint8, device="cuda"),
                           ooff=torch.arange(nb, dtype=torch.int64, device="cuda") * slot,
                           ocap=torch.full((nb,), slot, dtype=torch.int32, device="cuda"),
                           olen=torch.empty(nb, dtype=torch.int32, device="cuda"),
                           st=torch.empty(nb, dtype=torch.int32, device="cuda"))
        f = self._f
        st = _native.lib().lz4b200_compress_batch_device(
            ctx.handle, self.d_in.data_ptr(), f["off"].data_ptr(), f["len"].data_ptr(), f["flags"].data_ptr(),
            f["out"].data_ptr(), f["ooff"].data_ptr(), f["ocap"].data_ptr(), f["olen"].data_ptr(), f["st"].data_ptr(),
            nb, bs, torch.cuda.current_stream().cuda_stream)
        assert st == 0

    def verify(self, ctx):
        self.batch(ctx)
        torch.cuda.synchronize()
        bsid = int(self.info.block_size)
        want = [oracle.frame_compress(self.data[o:o + self.frame_len].tobytes(), bsid, self.flags) for o in self.off]
        offs = self.d_foff.cpu().numpy()
        assert offs.tolist() == np.cumsum([0] + [len(w) for w in want]).tolist()
        assert self.d_out[:int(offs[-1])].cpu().numpy().tobytes() == b"".join(want)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_compress_batch_device_probe"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    print("card:", card())
    ctx = block.Context(0)
    j = corpus.tiled("compression_66k_JSON.txt", GIB)
    h = corpus.tiled("hdfs.json", GIB)
    checks = oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM
    a = Case(j, 65536, FrameInfo(block_size=BlockSize.Max64KB), 0)
    b = Case(j, 65536, FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True), checks)
    c = Case(j, 4096, FrameInfo(block_size=BlockSize.Max64KB), 0)
    d = Case(h, 4 << 20, FrameInfo(block_size=BlockSize.Max4MB, block_checksums=True), oracle.F_BLOCK_CHECKSUMS)
    whole = Case(h, GIB, FrameInfo(block_size=BlockSize.Max4MB, block_checksums=True), oracle.F_BLOCK_CHECKSUMS)
    for x in (a, b, c, d):
        x.verify(ctx)
    print("outputs verified against the oracle")

    rows = {}
    runs = [("a batch", lambda: a.batch(ctx)), ("a compress_batch_device floor", lambda: a.floor(ctx)),
            ("a one-frame loop, per frame (512)", lambda: a.loop(ctx, 512)),
            ("b batch", lambda: b.batch(ctx)), ("b one-frame loop, per frame (512)", lambda: b.loop(ctx, 512)),
            ("c batch", lambda: c.batch(ctx)), ("c compress_batch_device floor", lambda: c.floor(ctx)),
            ("d batch", lambda: d.batch(ctx)), ("d one-frame call on the 1 GiB as one frame", lambda: whole.loop(ctx, 1))]
    for _, fn in runs:
        fn()
    for p in range(2):
        for name, fn in runs:
            t = timed(fn)
            if "per frame" in name:
                t /= 512
            rows.setdefault(name, []).append(round(t, 4))
    for name, x in (("a", a), ("c", c)):
        for p in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            x.batch(ctx)
            rows.setdefault(f"{name} batch, host time until the call returns", []).append(
                round((time.perf_counter() - t0) * 1e3, 4))
            torch.cuda.synchronize()
    for name, ts in rows.items():
        print(f"{name:45s} {ts} ms")
    kt = {}
    for name, fn in (("a", lambda: a.batch(ctx)), ("b", lambda: b.batch(ctx)), ("c", lambda: c.batch(ctx)),
                     ("d", lambda: d.batch(ctx))):
        kt[name] = kernel_times(fn, os.path.join(args.out, f"{name}.pt.trace.json"))
        print(name, json.dumps(kt[name]))
    with open(os.path.join(args.out, "frame_compress_batch_device_probe.json"), "w") as fh:
        json.dump({"card": card(), "times_ms": rows, "kernels_ms": kt}, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
