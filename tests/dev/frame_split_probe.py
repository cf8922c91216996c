"""Development aid: decoding concatenated frames in device memory, old per-frame loop against the split.

    python tests/dev/frame_split_probe.py [--out DIR] [--gib G]

Prints the card, its power limit and max SM clock.  For G GiB (default 1) of the JSON corpus compressed by
compress_frames_device as frames of 4 KiB, 64 KiB and 1 MiB, and by compress_frame_device as one frame, it checks the
new decode against the input and times (host clock to the end of a device synchronise, median of three after a warm-up):
  (a) the old per-frame loop: decompress_next_frame_device at d_in + consumed until the input ends;
  (b) decompress_frame_device (lz4b200_frame_decompress_device);
  (c) decompress_frames_device given the frame offsets and exact output offsets;
  (d) split_frames_device alone;
  (e) the old decoded bound (one lz4b200_frame_decoded_bound_device walk per frame, as the old call walked them) against
      the new decoded_bound_device.
The old loops (a) and (e) run over at most --loop-frames frames (default 4 096); when that is a prefix, the time per
frame and its product with the frame count are reported, marked as scaled.  Then the split of the converging-walks
input (split_cases.highway) at growing sizes, stopping after the first step that grows more than linearly."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import split_cases  # noqa: E402
from lz4_flex_b200 import block, corpus, frame  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return {"median_ms": statistics.median(ts) * 1e3, "min_ms": min(ts) * 1e3, "max_ms": max(ts) * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--gib", type=float, default=1.0)
    ap.add_argument("--loop-frames", type=int, default=4096)
    args = ap.parse_args()
    ctx = block.Context(0)
    total = int(args.gib * (1 << 30))
    raw = torch.from_numpy(corpus.tiled("compression_66k_JSON.txt", total).copy()).cuda()
    report = {"card": card(), "input_bytes": total, "cases": [], "highway": []}
    print(report["card"], flush=True)
    info = frame.FrameInfo(block_size=frame.BlockSize.Max64KB)
    for fsize in (4 << 10, 64 << 10, 1 << 20, None):
        if fsize is None:
            comp = frame.compress_frame_device(raw, frame.FrameInfo(block_size=frame.BlockSize.Max4MB), ctx=ctx)
            fo = np.array([0, comp.numel()], dtype=np.int64)
            name = "one frame"
        else:
            offs = np.arange(0, total, fsize, dtype=np.int64)
            comp, fo_t = frame.compress_frames_device(raw, offs, np.minimum(fsize, total - offs), info, ctx=ctx)
            fo = fo_t.cpu().numpy()
            name = f"{fsize >> 10} KiB frames"
        comp = comp.clone()
        F = len(fo) - 1
        out = torch.empty(total + 16, dtype=torch.uint8, device="cuda")
        got = frame.decompress_frame_device(comp, out, ctx)
        assert torch.equal(got, raw), name
        k = min(F, args.loop_frames)
        prefix = comp[:int(fo[k])]

        def old_loop():
            pos, w = 0, 0
            while pos < prefix.numel():
                used, n, err = frame.decompress_next_frame_device(prefix[pos:], out[w:], ctx)
                assert err is None
                w += n
                pos += used

        def old_bound():
            for i in range(k):
                frame.decoded_bound_device(comp[int(fo[i]):int(fo[i + 1])], ctx)

        fsz = np.diff(fo)
        contents = torch.tensor(np.minimum(fsize or total, total - np.arange(0, total, fsize or total)), device="cuda")
        ooff = torch.cumsum(contents, 0) - contents
        d_off, d_len = torch.tensor(fo[:-1], device="cuda"), torch.tensor(fsz, device="cuda")
        row = {"case": name, "frames": F, "compressed_bytes": int(fo[-1]), "loop_frames": k,
               "a_old_loop": timed(old_loop),
               "b_new": timed(lambda: frame.decompress_frame_device(comp, out, ctx)),
               "c_batch_with_offsets": timed(lambda: frame.decompress_frames_device(comp, d_off, d_len, out, ooff,
                                                                                     contents, ctx=ctx)),
               "d_split": timed(lambda: frame.split_frames_device(comp, ctx=ctx)),
               "e_old_bound": timed(old_bound),
               "e_new_bound": timed(lambda: frame.decoded_bound_device(comp, ctx))}
        if k < F:
            for key in ("a_old_loop", "e_old_bound"):
                row[key]["scaled_to_all_frames_ms"] = row[key]["median_ms"] * F / k
        report["cases"].append(row)
        print(json.dumps(row), flush=True)
        del comp, out
        torch.cuda.empty_cache()
    prev = None
    for blocks in (1 << 12, 1 << 14, 1 << 16, 1 << 18, 1 << 20):
        d = torch.from_numpy(np.frombuffer(split_cases.highway(blocks), np.uint8).copy()).cuda()
        t = timed(lambda: frame.split_frames_device(d, ctx=ctx))
        row = {"blocks": blocks, "bytes": d.numel(), "split": t}
        report["highway"].append(row)
        print(json.dumps(row), flush=True)
        if prev is not None and t["median_ms"] > 2 * 4 * prev:              # 4x the input: more than 8x the time
            break
        prev = t["median_ms"]
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "frame_split_probe.json"), "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
