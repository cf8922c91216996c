"""Development aid: the streaming device frame encoder (lz4b200_frame_encoder) against the one-shot device call
(lz4b200_frame_compress_device) on the same input, and the device memory each takes.

    python tests/dev/frame_encoder_device_probe.py [--out DIR] [--profile]

Prints the card and its power limit, then for
  (a) 1 GiB of 64 KiB JSON blocks, written in 1, 16 and 256 MiB pieces, at the default 256 MiB frame budget and at a
      budget that holds 21 blocks per SM (a full GPU of compress chains), without checksums and with block and content
      checksums;
  (b) 256 x 4 MiB hdfs blocks (1 GiB), written in 64 MiB pieces, at the default and at a 2 GiB budget;
the time of each (one checked warm-up, then two passes alternating with the one-shot call; host clock around a
sequence of calls that ends in a device synchronise; the calls themselves do not synchronise), the context's device
bytes after the run and the encoder's buffer.  With --profile, one extra pass of a few runs under torch.profiler gives
the summed CUDA time per kernel (buffer copy, plan, compress, scan and placement, gather, block checksum, content
hash)."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from lz4_flex_b200 import _native, block, corpus  # noqa: E402
from lz4_flex_b200.frame import BlockSize, FrameInfo  # noqa: E402

WRITE, FINISH = 0, 2


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def slot(n):
    return (20 + n * 110 // 100 + 15) & ~15


def one_shot(ctx, d_in, info, out, d_w):
    ci = info.to_c()
    st = _native.lib().lz4b200_frame_compress_device(ctx.handle, d_in.data_ptr(), d_in.numel(), C.byref(ci),
                                                     d_in.numel(), out.data_ptr(), out.numel(), d_w.data_ptr(),
                                                     torch.cuda.current_stream().cuda_stream)
    assert st == 0, st


class Streamed:
    """One encoder on its own context; a pass writes d_in in pieces and finishes, each call's output in a region of
    its bound, without a synchronise between calls."""

    def __init__(self, info, budget, piece, n):
        L = _native.lib()
        self.ctx = block.Context(0)
        if budget:
            L.lz4b200_ctx_set_frame_budget(self.ctx.handle, budget)
        self.budget = budget or (256 << 20)
        ci = info.to_c()
        self.h = C.c_void_p()
        assert L.lz4b200_frame_encoder_create(self.ctx.handle, C.byref(ci), C.byref(self.h)) == 0
        self.info, self.piece = info, piece
        self.ncalls = -(-n // piece) + 1
        self.out = torch.empty(n + n // 64 + 4096 * self.ncalls + (16 << 20), dtype=torch.uint8, device="cuda")
        self.lens = torch.empty(self.ncalls, dtype=torch.int64, device="cuda")

    def run(self, d_in):
        L = _native.lib()
        s = torch.cuda.current_stream().cuda_stream
        pos, regions = 0, []
        n = d_in.numel()
        for i, a in enumerate(list(range(0, n, self.piece)) + [n]):
            m = min(self.piece, n - a)
            op = FINISH if a == n else WRITE
            b = L.lz4b200_frame_encoder_bound(self.h, m, op)
            assert pos + b <= self.out.numel()
            st = L.lz4b200_frame_encoder_encode_device(self.h, d_in[a:].data_ptr() if m else None, m, op,
                                                       self.out[pos:].data_ptr(), b, self.lens[i:].data_ptr(), s)
            assert st == 0, st
            regions.append(pos)
            pos += b
        return regions

    def frame(self, regions):
        lens = self.lens.cpu().tolist()
        return torch.cat([self.out[p:p + w] for p, w in zip(regions, lens)])

    def device_bytes(self):
        bs = self.info.block_size.get_size()
        group = max(1, self.budget // (bs + slot(bs)))
        return int(_native.lib().lz4b200_ctx_device_bytes(self.ctx.handle)), group, group * bs

    def close(self):
        _native.lib().lz4b200_frame_encoder_destroy(self.h)
        self.ctx.close()


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def measure(name, d_in, info, configs, rows):
    """configs: [(label, budget or None, piece)]."""
    n = d_in.numel()
    one_ctx = block.Context(0)
    ci = info.to_c()
    full = torch.empty(_native.lib().lz4b200_frame_bound(n, C.byref(ci)), dtype=torch.uint8, device="cuda")
    d_w = torch.empty(1, dtype=torch.int64, device="cuda")
    one_shot(one_ctx, d_in, info, full, d_w)
    want = full[:int(d_w.item())].clone()
    runs = {}
    for label, budget, piece in configs:
        r = Streamed(info, budget, piece, n)
        got = r.frame(r.run(d_in))
        assert torch.equal(got, want), label                              # the same frame as the one-shot call
        runs[label] = r
    times = {k: [] for k in ["one-shot"] + list(runs)}
    for _ in range(2):
        times["one-shot"].append(timed(lambda: one_shot(one_ctx, d_in, info, full, d_w)))
        for label, r in runs.items():
            times[label].append(timed(lambda: r.run(d_in)))
    row = {"input": name, "run": "one-shot", "ms": [round(t, 1) for t in times["one-shot"]],
           "ctx_device_bytes": int(_native.lib().lz4b200_ctx_device_bytes(one_ctx.handle))}
    rows.append(row)
    print(json.dumps(row), flush=True)
    for label, r in runs.items():
        cb, group, buf = r.device_bytes()
        row = {"input": name, "run": label, "ms": [round(t, 1) for t in times[label]], "calls": r.ncalls,
               "group_blocks": group, "ctx_device_bytes": cb, "encoder_buffer_bytes": buf}
        rows.append(row)
        print(json.dumps(row), flush=True)
    return one_ctx, runs


def profile(name, d_in, info, budget, piece, rows):
    from torch.profiler import ProfilerActivity, profile as tprofile
    r = Streamed(info, budget, piece, d_in.numel())
    r.run(d_in)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        r.run(d_in)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        key = ev.name[:60]
        per[key] = per.get(key, 0.0) + ev.time_range.elapsed_us() / 1e3
    row = {"input": name, "profile": f"budget {budget or 256 << 20}, {piece >> 20} MiB pieces",
           "kernel_ms": {k: round(v, 2) for k, v in sorted(per.items(), key=lambda kv: -kv[1]) if v >= 0.01}}
    rows.append(row)
    print(json.dumps(row), flush=True)
    r.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    rows = [{"card": card(), "sm_count": torch.cuda.get_device_properties(0).multi_processor_count}]
    print(json.dumps(rows[0]), flush=True)
    sms = rows[0]["sm_count"]
    full_gpu = 21 * sms * (65536 + slot(65536))                          # 21 chains per SM, one 64 KiB block each

    j = torch.from_numpy(corpus.tiled("compression_66k_JSON.txt", 1 << 30)).cuda()
    for checks in (False, True):
        info = FrameInfo(block_size=BlockSize.Max64KB, block_checksums=checks, content_checksum=checks)
        configs = [(f"{p} MiB pieces, budget {'default' if b is None else f'{b >> 20} MiB'}", b, p << 20)
                   for b in (None, full_gpu) for p in (1, 16, 256)]
        one_ctx, runs = measure(f"1 GiB JSON 64 KiB blocks{', checksums' if checks else ''}", j, info, configs, rows)
        for r in runs.values():
            r.close()
        one_ctx.close()
    h = torch.from_numpy(corpus.tiled("hdfs.json", 1 << 30)).cuda()
    info = FrameInfo(block_size=BlockSize.Max4MB, block_checksums=True)
    one_ctx, runs = measure("256 x 4 MiB hdfs blocks, block checksums", h, info,
                            [("64 MiB pieces, budget default", None, 64 << 20),
                             ("64 MiB pieces, budget 2048 MiB", 2048 << 20, 64 << 20)], rows)
    for r in runs.values():
        r.close()
    one_ctx.close()
    if args.profile:
        profile("1 GiB JSON 64 KiB blocks", j, FrameInfo(block_size=BlockSize.Max64KB), None, 16 << 20, rows)
        profile("1 GiB JSON 64 KiB blocks, checksums", j,
                FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True), None, 16 << 20, rows)
        profile("256 x 4 MiB hdfs blocks", h, FrameInfo(block_size=BlockSize.Max4MB), None, 64 << 20, rows)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        json.dump(rows, open(os.path.join(args.out, "frame_encoder_device_probe.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
