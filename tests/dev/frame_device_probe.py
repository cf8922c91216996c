"""Development aid: the device-resident frame decoder (lz4b200_frame_decompress_next_device) against the host frame
decoder (lz4b200_frame_decompress_next) and the block-batch floor (lz4b200_decompress_batch_device) on the same blocks.

    python tests/dev/frame_device_probe.py [--out DIR] [--gib 1]

Prints the card and its power limit, checks every output against the input, then for three frames
  (a) 1 GiB of 64 KiB JSON blocks, no checksums; (b) the same with block and content checksums;
  (c) 256 x 4 MiB hdfs blocks
times the three calls (one warm-up, then two alternating passes; host clock around calls that end in a device
synchronise).  A separate profiled call per frame gives the device time of the walk, block-checksum, content-hash,
decode and gather kernels (torch.profiler).  Finally one profiled device decode of a 64 MiB frame with block and
content checksums lists every host<->device copy, to show that no payload crosses PCIe."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from lz4_flex_b200 import _native, block, corpus, frame  # noqa: E402
from lz4_flex_b200.frame import BlockSize, FrameInfo  # noqa: E402

KERNELS = ("frame_walk_kernel", "block_checksum_kernel", "content_hash_kernel", "lz4_decompress_blocks", "gather_segments_kernel")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def blocks_of(f: bytes, bs: int):
    """(payload offsets, lengths, decoded offsets, stored flags) of a frame's blocks, from its BlockInfo words."""
    flg = f[4]
    pos = 7 + (8 if flg & 0x08 else 0)
    offs, lens, stored = [], [], []
    while True:
        w = int.from_bytes(f[pos:pos + 4], "little")
        pos += 4
        if w == 0:
            break
        offs.append(pos); lens.append(w & 0x7FFFFFFF); stored.append(bool(w >> 31))
        pos += (w & 0x7FFFFFFF) + (4 if flg & 0x10 else 0)
    return np.array(offs), np.array(lens), np.array(stored)


def host_next(ctx, src: np.ndarray, out: np.ndarray):
    used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
    st = _native.lib().lz4b200_frame_decompress_next(ctx.handle, src.ctypes.data, src.size, out.ctypes.data, out.size,
                                                     C.byref(used), C.byref(w), C.byref(bs), C.byref(e1), C.byref(e2))
    assert st == 0, st
    return w.value


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def kernel_times(fn, trace_path=None):
    """Device time per kernel family (ms) and the host<->device copies of one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = trace_path or os.path.join(tempfile.gettempdir(), "frame_device_probe.trace.json")
    prof.export_chrome_trace(path)
    ev = json.load(open(path))["traceEvents"]
    k = {name: [0, 0.0] for name in KERNELS}
    copies = []
    for e in ev:
        if e.get("cat") == "kernel":
            for name in KERNELS:
                if name in e["name"]:
                    k[name][0] += 1
                    k[name][1] += e["dur"] / 1e3
        elif e.get("cat") == "gpu_memcpy":
            copies.append((e["name"], int(e.get("args", {}).get("bytes", -1))))
    return k, copies


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_device_probe"),
                    help="directory for the profiler trace of the 64 MiB decode")
    ap.add_argument("--gib", type=float, default=1.0)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    print("card:", card(), flush=True)
    ctx = block.Context(0)
    total = int(args.gib * (1 << 30))
    json_data = corpus.tiled("compression_66k_JSON.txt", total)
    hdfs = corpus.tiled("hdfs.json", 256 << 22)
    cases = [
        ("a: 64 KiB JSON blocks, no checksums", json_data, FrameInfo(block_size=BlockSize.Max64KB)),
        ("b: 64 KiB JSON blocks, block + content checksums", json_data,
         FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True)),
        ("c: 256 x 4 MiB hdfs blocks", hdfs, FrameInfo(block_size=BlockSize.Max4MB)),
    ]
    rows = []
    for name, data, info in cases:
        f = frame.compress_frame(data, info, ctx)
        src = np.frombuffer(f, dtype=np.uint8)
        d_in = torch.from_numpy(src.copy()).cuda()
        d_out = torch.empty(data.size, dtype=torch.uint8, device="cuda")
        h_out = np.empty(data.size, dtype=np.uint8)
        want = torch.from_numpy(data).cuda()
        offs, lens, stored = blocks_of(f, info.block_size.get_size())
        assert not stored.any()
        bsz = info.block_size.get_size()
        batch = block.DeviceBatch(offs, lens, np.arange(len(lens), dtype=np.uint64) * bsz, np.full(len(lens), bsz))
        d_floor = torch.empty(data.size, dtype=torch.uint8, device="cuda")

        def dev():
            used, w, err = frame.decompress_next_frame_device(d_in, d_out, ctx)
            assert err is None and used == len(f) and w == data.size, (used, w, err)

        def host():
            assert host_next(ctx, src, h_out) == data.size

        def floor():
            batch.decompress(d_in, d_floor, ctx)

        dev(); host(); floor()                                                   # warm-up, and the outputs checked
        torch.cuda.synchronize()
        assert torch.equal(d_out, want), name
        assert np.array_equal(h_out, data), name
        assert torch.equal(d_floor, want) and not batch.status.any(), name
        t = {"device": [], "host": [], "floor": []}
        for _ in range(2):
            t["device"].append(timed(dev)); t["host"].append(timed(host)); t["floor"].append(timed(floor))
        k, _ = kernel_times(dev)
        row = {"frame": name, "frame_bytes": len(f), "decoded_bytes": int(data.size), "blocks": int(len(lens)),
               "ms": {n: [round(v, 2) for v in vs] for n, vs in t.items()},
               "kernels_ms": {n: {"launches": c, "ms": round(ms, 3)} for n, (c, ms) in k.items()}}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del d_in, d_out, d_floor, want, batch
        torch.cuda.empty_cache()

    # ---- no payload crosses PCIe: every copy of one device decode of a 64 MiB frame with both checksums -------------------
    data = corpus.tiled("compression_66k_JSON.txt", 64 << 20)
    f = frame.compress_frame(data, FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True), ctx)
    d_in = torch.from_numpy(np.frombuffer(f, dtype=np.uint8).copy()).cuda()
    d_out = torch.empty(data.size, dtype=torch.uint8, device="cuda")
    frame.decompress_next_frame_device(d_in, d_out, ctx)
    k, copies = kernel_times(lambda: frame.decompress_next_frame_device(d_in, d_out, ctx),
                             os.path.join(args.out, "frame_device_64mib.pt.trace.json"))
    assert torch.equal(d_out, torch.from_numpy(data).cuda())
    nblocks = (64 << 20) // 65536
    summary = {}
    for n, b in copies:
        s = summary.setdefault(n, {"count": 0, "bytes": 0, "largest": 0})
        s["count"] += 1; s["bytes"] += b; s["largest"] = max(s["largest"], b)
    print(json.dumps({"trace_64mib": {"frame_bytes": len(f), "blocks": nblocks, "descriptor_bytes": 16 * nblocks,
                                      "copies": summary,
                                      "kernels_ms": {n: {"launches": c, "ms": round(ms, 3)} for n, (c, ms) in k.items()}}}),
          flush=True)
    largest = max((b for _, b in copies), default=0)
    assert largest <= 16 * nblocks, f"a copy of {largest} bytes crossed PCIe"
    print("ok")


if __name__ == "__main__":
    main()
