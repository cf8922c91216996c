"""Development aid: the linked batch frame encoder (lz4b200_frame_compress_linked_batch_device) against the independent
batch frame encoder (lz4b200_frame_compress_batch_device) on the same inputs.

    python tests/dev/frame_linked_compress_probe.py [--out DIR] [--cpu-only]

Prints the card and its power limit, then
  (a) one linked frame of dickens (the whole 10 MB file, 64 KiB blocks): the rate of one chain;
  (b) batches of 1, 132, 1 584 and 16 384 frames of 64 KiB and of 1 MiB inputs (JSON and dickens, 64 KiB blocks):
      linked against independent, each timed with device events after a warm-up (median of three calls);
  (c) the linked / independent frame size ratio, from the CPU references (tests/cpp/linked_frame_ref.c and the C
      oracle): a CPU number, it needs no GPU.
The first, middle and last GPU frame of the first call of each case are compared with the CPU reference's.  Batches whose input would exceed
4 GiB are skipped and reported as not measured.  Results go to DIR/frame_linked_compress_probe.json as well."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import linked_ref  # noqa: E402
import oracle  # noqa: E402
from lz4_flex_b200 import corpus  # noqa: E402



def ratios():
    out = {}
    dk = corpus.load("dickens.txt")
    js = corpus.tiled("compression_66k_JSON.txt", len(dk)).tobytes()
    for name, d in (("dickens", dk), ("json", js)):
        for bsid, bsn in ((4, "64K"), (6, "1M")):
            ind, lnk = len(oracle.frame_compress(d, bsid, 0)), len(linked_ref.frame_compress(d, bsid))
            out[f"{name} {bsn} blocks"] = {"independent": ind, "linked": lnk, "linked/independent": round(lnk / ind, 4)}
    return out


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    import torch
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def time_call(fn, reps=3):
    import torch
    fn()                                                    # warm-up (and the call whose output is checked)
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def gpu_cases(ctx):
    import torch
    from lz4_flex_b200 import frame
    from lz4_flex_b200.frame import BlockMode, BlockSize, FrameInfo
    lnk_info = FrameInfo(block_size=BlockSize.Max64KB, block_mode=BlockMode.Linked)
    ind_info = FrameInfo(block_size=BlockSize.Max64KB)
    dk = corpus.load("dickens.txt")
    res = {}

    # (a) one chain
    d_in = torch.tensor(np.frombuffer(dk, dtype=np.uint8), device="cuda")
    out, offs = frame.compress_linked_frames_device(d_in, [0], [len(dk)], lnk_info, ctx=ctx)
    assert out.cpu().numpy().tobytes() == linked_ref.frame_compress(dk, 4), "the frame differs from the reference"
    ms = time_call(lambda: frame.compress_linked_frames_device(d_in, [0], [len(dk)], lnk_info, ctx=ctx))
    res["one linked frame, dickens 9.99 MB, 64 KiB blocks"] = {"ms": round(ms, 2), "MB/s": round(len(dk) / ms / 1e3, 1)}
    print(json.dumps(res), flush=True)

    # (b) batches
    for src_name in ("json", "dickens"):
        for size in (64 << 10, 1 << 20):
            for n in (1, 132, 1584, 16384):
                key = f"{n} x {size >> 10} KiB {src_name}"
                if n * size > 4 << 30:
                    res[key] = "not measured"
                    continue
                if src_name == "json":
                    flat = corpus.tiled("compression_66k_JSON.txt", n * size)
                    starts = np.arange(n, dtype=np.int64) * size
                    host = flat
                    d_in = torch.tensor(host, device="cuda")
                else:
                    starts = (np.arange(n, dtype=np.int64) * 33331) % (len(dk) - size)
                    host = np.frombuffer(dk, dtype=np.uint8)
                    d_in = torch.tensor(host, device="cuda")
                lens = np.full(n, size, dtype=np.int64)
                row = {}
                for name, fn, info, ref in (("linked", frame.compress_linked_frames_device, lnk_info,
                                             lambda d: linked_ref.frame_compress(d, 4)),
                                            ("independent", frame.compress_frames_device, ind_info,
                                             lambda d: oracle.frame_compress(d, 4, 0))):
                    out, offs = fn(d_in, starts, lens, info, ctx=ctx)
                    o = offs.cpu().numpy()
                    h = out.cpu().numpy().tobytes()
                    for i in sorted({0, n // 2, n - 1}):
                        d = host[starts[i]:starts[i] + size].tobytes()
                        assert h[o[i]:o[i + 1]] == ref(d), (key, name, i)
                    ms = time_call(lambda: fn(d_in, starts, lens, info, ctx=ctx))
                    row[name] = {"ms": round(ms, 3), "GB/s": round(n * size / ms / 1e6, 3)}
                row["linked/independent time"] = round(row["linked"]["ms"] / row["independent"]["ms"], 2)
                res[key] = row
                print(key, json.dumps(row), flush=True)
                del d_in
                torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--cpu-only", action="store_true", help="the CPU references' size ratios alone")
    a = ap.parse_args()
    rec = {"size ratio (CPU references)": ratios()}
    print(json.dumps(rec["size ratio (CPU references)"], indent=1), flush=True)
    if not a.cpu_only:
        from lz4_flex_b200 import block
        rec["card"] = card()
        print("card:", rec["card"], flush=True)
        ctx = block.Context(0)
        try:
            rec["gpu"] = gpu_cases(ctx)
        finally:
            ctx.close()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "frame_linked_compress_probe.json"), "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
