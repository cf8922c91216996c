"""Development aid: the frame index (lz4b200_frame_index_device) and the range decoder
(lz4b200_frame_decompress_ranges_device) against a whole-frame decode (lz4b200_frame_decompress_next_device).

    python tests/dev/frame_range_probe.py [--out DIR] [--profile]

Prints the card and its power limit, checks every output against the source, then for
  (a) a 1 GiB frame of 64 KiB JSON blocks and (b) a 256 MiB frame of 4 MiB hdfs blocks: the index build against the
      whole-frame decode, and range calls of 10 000 x 4 KiB and 100 x 1 MiB random ranges;
  (c) tests/golden/linked/json_1m_256k_linked.lz4: index, whole-frame decode, and 100 x 4 KiB ranges (a linked frame
      decodes from its first block up to the furthest range)
times each call (one warm-up, then three alternating passes; host clock around calls that end in a device
synchronise).  With --profile, one profiled call per case gives the device time of each kernel (torch.profiler)."""
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
from lz4_flex_b200 import block, corpus, frame  # noqa: E402


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


def cases():
    j = torch.tensor(corpus.tiled("compression_66k_JSON.txt", 1 << 30), device="cuda")
    h = torch.tensor(corpus.tiled("hdfs.json", 256 << 20), device="cuda")
    out = [("json 1 GiB / 64 KiB", j, frame.compress_frame_device(j, frame.FrameInfo(block_size=frame.BlockSize.Max64KB))),
           ("hdfs 256 MiB / 4 MiB", h, frame.compress_frame_device(h, frame.FrameInfo(block_size=frame.BlockSize.Max4MB)))]
    lf = open(os.path.join(ROOT, "tests", "golden", "linked", "json_1m_256k_linked.lz4"), "rb").read()
    d = torch.tensor(np.frombuffer(lf, dtype=np.uint8), device="cuda")
    out.append(("linked json 1 MiB / 256 KiB", frame.decompress_frame_device(d), d))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_range_probe"))
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    ctx = block.Context(0)
    rng = np.random.default_rng(1)
    rec = {"card": card(), "cases": []}
    print(rec["card"], flush=True)
    for name, src, f in cases():
        n = src.numel()
        idx = frame.index_frame_device(f, ctx)
        assert idx.error is None and idx.content_len == n, name
        whole = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
        sets = {}
        for count, size in ((10000, 4096), (100, 1 << 20)):
            if size * count > n * 4:                     # the small linked frame: 100 ranges per call
                count = 100
            label = f"{count} x {size >> 10} KiB"
            st = rng.integers(0, max(n - size, 1), count)
            ln = np.full(count, min(size, n))
            out, oo, _ = frame.decompress_ranges_device(f, idx, st, ln, ctx=ctx)
            within = np.arange(int(ln.sum())) - np.repeat(np.cumsum(ln) - ln, ln)
            assert torch.equal(out[torch.as_tensor(np.repeat(oo.cpu().numpy(), ln) + within, device="cuda")],
                               src[torch.as_tensor(np.repeat(st, ln) + within, device="cuda")]), (name, label)
            sets[label] = (st, ln, out, oo)
        calls = {"index": lambda: frame.index_frame_device(f, ctx),
                 "whole-frame decode": lambda: frame.decompress_next_frame_device(f, whole, ctx)}
        for label, (st, ln, out, oo) in sets.items():
            ts, tl = torch.as_tensor(st, device="cuda"), torch.as_tensor(ln, device="cuda")
            calls[f"ranges {label}"] = (lambda ts=ts, tl=tl, out=out, oo=oo:
                                        frame.decompress_ranges_device(f, idx, ts, tl, out=out, out_offsets=oo, ctx=ctx))
        for fn in calls.values():
            fn()
        times = {k: [] for k in calls}
        for _ in range(3):
            for k, fn in calls.items():
                times[k].append(timed(fn))
        r = {"case": name, "content": n, "blocks": idx.nblocks, "ms": {k: sorted(v) for k, v in times.items()}}
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            prof_rows = {}
            for k, fn in calls.items():
                with profile(activities=[ProfilerActivity.CUDA]) as p:
                    fn()
                    torch.cuda.synchronize()
                prof_rows[k] = {e.key: round(e.device_time_total / 1e3, 3) for e in p.key_averages()
                                if e.device_time_total > 0}
            r["kernels_ms"] = prof_rows
        rec["cases"].append(r)
        print(json.dumps(r), flush=True)
    with open(os.path.join(a.out, "frame_range_probe.json"), "w") as fh:
        json.dump(rec, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
