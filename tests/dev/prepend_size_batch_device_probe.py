"""Development aid: the size-prepended batch calls (lz4b200_compress_prepend_size_batch_device,
lz4b200_decompress_size_prepended_batch_device) against their floors, the block batch calls on the same blocks
(lz4b200_compress_batch_device into one slot per block, lz4b200_decompress_batch_device from the records' blocks into
a layout computed on the host).

    python tests/dev/prepend_size_batch_device_probe.py [--out DIR]

Prints the card, its power limit and max SM clock, checks every record against the floor's blocks, a sample against
the C oracle, and the round trip against the input, then for
  (a) 16 384 records of 64 KiB JSON (1 GiB);
  (b) 262 144 records of 4 KiB JSON (1 GiB);
  (c) 256 records of 4 MiB hdfs (1 GiB)
times each call (one warm-up, then two alternating passes; host clock around calls that end in a device synchronise),
and the host time until each size-prepended call returns (after a synchronise).  A separate profiled call per case and
direction gives the device time of each kernel (torch.profiler)."""
import argparse
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

GIB = 1 << 30


class Case:
    def __init__(self, data: np.ndarray, bs: int):
        L = _native.lib()
        self.n, self.bs, self.data = data.size // bs, bs, data
        n = self.n
        self.d_in = torch.from_numpy(data).cuda()
        self.in_off = torch.arange(n, dtype=torch.int64, device="cuda") * bs
        self.in_len = torch.full((n,), bs, dtype=torch.int32, device="cuda")
        self.cap = n * (4 + L.lz4b200_max_output_size(bs))
        self.recs = torch.empty(self.cap, dtype=torch.uint8, device="cuda")
        self.rec_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        self.cstatus = torch.empty(n, dtype=torch.int32, device="cuda")
        self.dec = torch.empty(n * bs, dtype=torch.uint8, device="cuda")
        self.out_off = torch.empty(n + 1, dtype=torch.int64, device="cuda")
        self.out_len = torch.empty(n, dtype=torch.int32, device="cuda")
        self.dstatus = torch.empty(n, dtype=torch.int32, device="cuda")
        self.expected = torch.empty(n, dtype=torch.int64, device="cuda")
        slot = L.lz4b200_max_output_size(bs)
        self.f = dict(out=torch.empty(n * slot, dtype=torch.uint8, device="cuda"),
                      ooff=torch.arange(n, dtype=torch.int64, device="cuda") * slot,
                      ocap=torch.full((n,), slot, dtype=torch.int32, device="cuda"),
                      olen=torch.empty(n, dtype=torch.int32, device="cuda"),
                      st=torch.empty(n, dtype=torch.int32, device="cuda"),
                      dec=torch.empty(n * bs, dtype=torch.uint8, device="cuda"),
                      doff=torch.arange(n, dtype=torch.int64, device="cuda") * bs,
                      dlen=torch.empty(n, dtype=torch.int32, device="cuda"),
                      dexp=torch.empty(n, dtype=torch.int64, device="cuda"))

    def compress(self, ctx):
        st = _native.lib().lz4b200_compress_prepend_size_batch_device(
            ctx.handle, self.d_in.data_ptr(), self.in_off.data_ptr(), self.in_len.data_ptr(), self.n, self.bs,
            self.recs.data_ptr(), self.cap, self.rec_off.data_ptr(), self.cstatus.data_ptr(),
            torch.cuda.current_stream().cuda_stream)
        assert st == 0, ctx.last_cuda_error()

    def decompress(self, ctx):
        st = _native.lib().lz4b200_decompress_size_prepended_batch_device(
            ctx.handle, self.recs.data_ptr(), self.rec_off.data_ptr(), self.rec_len.data_ptr(), self.n,
            self.dec.data_ptr(), self.dec.numel(), self.out_off.data_ptr(), self.out_len.data_ptr(),
            self.dstatus.data_ptr(), self.expected.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert st == 0, ctx.last_cuda_error()

    def floor_compress(self, ctx):
        f = self.f
        st = _native.lib().lz4b200_compress_batch_device(
            ctx.handle, self.d_in.data_ptr(), self.in_off.data_ptr(), self.in_len.data_ptr(), None, f["out"].data_ptr(),
            f["ooff"].data_ptr(), f["ocap"].data_ptr(), f["olen"].data_ptr(), f["st"].data_ptr(), self.n, self.bs,
            torch.cuda.current_stream().cuda_stream)
        assert st == 0

    def floor_decompress(self, ctx):
        """The records' blocks, with the output layout the host computed beforehand."""
        f = self.f
        st = _native.lib().lz4b200_decompress_batch_device(
            ctx.handle, self.recs.data_ptr(), self.blk_off.data_ptr(), self.blk_len.data_ptr(), f["dec"].data_ptr(),
            f["doff"].data_ptr(), self.in_len.data_ptr(), f["dlen"].data_ptr(), f["st"].data_ptr(), f["dexp"].data_ptr(),
            self.n, torch.cuda.current_stream().cuda_stream)
        assert st == 0

    def verify(self, ctx):
        self.compress(ctx)
        self.floor_compress(ctx)
        torch.cuda.synchronize()
        assert (self.cstatus == 0).all().item() and (self.f["st"] == 0).all().item()
        self.rec_len = (self.rec_off[1:] - self.rec_off[:-1]).to(torch.int32)
        self.blk_off, self.blk_len = self.rec_off[:-1] + 4, self.rec_len - 4
        assert torch.equal(self.blk_len, self.f["olen"])
        ro = self.rec_off.cpu().numpy()
        recs, blocks = self.recs[:int(ro[-1])].cpu().numpy(), self.f["out"].cpu().numpy()
        slot = _native.lib().lz4b200_max_output_size(self.bs)
        for b in range(self.n):
            assert recs[ro[b]:ro[b] + 4].tobytes() == self.bs.to_bytes(4, "little")
            assert recs[ro[b] + 4:ro[b + 1]].tobytes() == blocks[b * slot:b * slot + ro[b + 1] - ro[b] - 4].tobytes()
        for b in np.random.default_rng(0).integers(0, self.n, 32):
            assert recs[ro[b]:ro[b + 1]].tobytes() == oracle.compress_prepend_size(self.data[b * self.bs:(b + 1) * self.bs])
        self.decompress(ctx)
        self.floor_decompress(ctx)
        torch.cuda.synchronize()
        assert (self.dstatus == 0).all().item() and (self.f["st"] == 0).all().item()
        assert torch.equal(self.dec, self.d_in) and torch.equal(self.f["dec"], self.d_in)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "prepend_size_batch_device_probe"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    print("card:", card())
    ctx = block.Context(0)
    rows, kt = {}, {}
    specs = [("a", "compression_66k_JSON.txt", 65536), ("b", "compression_66k_JSON.txt", 4096), ("c", "hdfs.json", 4 << 20)]
    for name, src, bs in specs:
        c = Case(corpus.tiled(src, GIB), bs)
        c.verify(ctx)
        print(f"{name}: {c.n} records of {bs} B verified, ratio {int(c.rec_off[-1]) / GIB:.3f}")
        runs = [("compress_prepend_size_batch_device", lambda: c.compress(ctx)),
                ("compress_batch_device floor", lambda: c.floor_compress(ctx)),
                ("decompress_size_prepended_batch_device", lambda: c.decompress(ctx)),
                ("decompress_batch_device floor", lambda: c.floor_decompress(ctx))]
        for _, fn in runs:
            fn()
        for _ in range(2):
            for what, fn in runs:
                rows.setdefault(f"{name} {what}", []).append(round(timed(fn), 3))
        for what, fn in runs[::2]:
            for _ in range(2):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                rows.setdefault(f"{name} {what}, host time until it returns", []).append(
                    round((time.perf_counter() - t0) * 1e3, 4))
                torch.cuda.synchronize()
        for what, fn in runs[::2]:
            kt[f"{name} {what}"] = kernel_times(fn, os.path.join(args.out, f"{name}_{what}.pt.trace.json"))
            print(name, what, json.dumps(kt[f"{name} {what}"]))
        del c
        torch.cuda.empty_cache()
    for name, ts in rows.items():
        print(f"{name:70s} {ts} ms")
    with open(os.path.join(args.out, "prepend_size_batch_device_probe.json"), "w") as fh:
        json.dump({"card": card(), "times_ms": rows, "kernels_ms": kt}, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
