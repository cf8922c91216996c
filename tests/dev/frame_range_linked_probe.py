"""Development aid: ranges of linked frames (lz4b200_frame_decompress_ranges_device, marker decode from a look-back)
against a whole-frame decode (lz4b200_frame_decompress_next_device).

    python tests/dev/frame_range_linked_probe.py [--out DIR] [--profile]

Prints the card and its power limit, checks every output against the source, then for linked frames built by
tests/stream_frames.linked_frame (256 MiB JSON in 64 KiB blocks, 256 MiB hdfs in 4 MiB blocks, dickens in 64 KiB blocks,
a random 60 KiB pattern repeated over 64 MiB in 64 KiB blocks) and tests/golden/linked/json_1m_256k_linked.lz4 times the
whole-frame decode, one 4 KiB range near the start and one near the end, 10 000 x 4 KiB and 100 x 1 MiB random ranges,
with the block decodes lz4b200_ctx_last_range_blocks reports for each (one warm-up, then three alternating passes; host
clock around calls that end in a device synchronise).  With --profile, one profiled call per case gives the device
time of each kernel (torch.profiler)."""
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
from lz4_flex_b200 import _native, block, corpus, frame  # noqa: E402
from stream_frames import linked_frame  # noqa: E402

MiB = 1 << 20


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
    rnd = np.random.default_rng(5).integers(0, 256, 60 << 10, dtype=np.uint8).tobytes()
    srcs = [("json 256 MiB / 64 KiB", corpus.tiled("compression_66k_JSON.txt", 256 * MiB).tobytes(), 65536, 4),
            ("hdfs 256 MiB / 4 MiB", corpus.tiled("hdfs.json", 256 * MiB).tobytes(), 4 * MiB, 7),
            ("dickens / 64 KiB", corpus.load("dickens.txt"), 65536, 4),
            ("random 60 KiB x 1118 / 64 KiB", rnd * 1118, 65536, 4)]
    for name, data, bl, bsid in srcs:
        f = linked_frame(data, [bl], bsid=bsid)
        yield name, torch.tensor(np.frombuffer(data, dtype=np.uint8), device="cuda"), \
            torch.tensor(np.frombuffer(f, dtype=np.uint8), device="cuda")
    lf = open(os.path.join(ROOT, "tests", "golden", "linked", "json_1m_256k_linked.lz4"), "rb").read()
    d = torch.tensor(np.frombuffer(lf, dtype=np.uint8), device="cuda")
    yield "golden json 1 MiB / 256 KiB", frame.decompress_frame_device(d), d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_range_linked_probe"))
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
        assert idx.error is None and idx.linked and idx.content_len == n, name
        whole = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
        sets = {"4 KiB at start": (np.array([4096]), np.array([4096])),
                "4 KiB at end": (np.array([n - 8192]), np.array([4096]))}
        for count, size in ((10000, 4096), (100, MiB)):
            count = min(count, max(n // size, 1) * 4)
            sets[f"{count} x {size >> 10} KiB"] = (rng.integers(0, max(n - size, 1), count), np.full(count, min(size, n)))
        calls, blocks = {"whole-frame decode": lambda: frame.decompress_next_frame_device(f, whole, ctx)}, {}
        for label, (st, ln) in sets.items():
            out, oo, _ = frame.decompress_ranges_device(f, idx, st, ln, ctx=ctx)
            blocks[label] = int(_native.lib().lz4b200_ctx_last_range_blocks(ctx.handle))
            within = np.arange(int(ln.sum())) - np.repeat(np.cumsum(ln) - ln, ln)
            assert torch.equal(out[torch.as_tensor(np.repeat(oo.cpu().numpy(), ln) + within, device="cuda")],
                               src[torch.as_tensor(np.repeat(st, ln) + within, device="cuda")]), (name, label)
            ts, tl = torch.as_tensor(st, device="cuda"), torch.as_tensor(ln, device="cuda")
            calls[f"ranges {label}"] = (lambda ts=ts, tl=tl, out=out, oo=oo:
                                        frame.decompress_ranges_device(f, idx, ts, tl, out=out, out_offsets=oo, ctx=ctx))
        for fn in calls.values():
            fn()
        times = {k: [] for k in calls}
        for _ in range(3):
            for k, fn in calls.items():
                times[k].append(round(timed(fn), 3))
        r = {"case": name, "content": n, "blocks": idx.nblocks, "ms": {k: sorted(v) for k, v in times.items()},
             "block_decodes": blocks}
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
    with open(os.path.join(a.out, "frame_range_linked_probe.json"), "w") as fh:
        json.dump(rec, fh, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
