"""Development aid: the device-resident frame encoder (lz4b200_frame_compress_device) against the host frame encoder
(lz4b200_frame_compress, input and output in pinned host memory) and the block-range floor
(lz4b200_frame_compress_blocks_device: the same blocks, no header, EndMark or checksums).

    python tests/dev/frame_compress_device_probe.py [--out DIR] [--gib 1]

Prints the card, its power limit and its max SM clock, checks every device frame against the host call, then for three
frames
  (a) 1 GiB of 64 KiB JSON blocks, no checksums; (b) the same with block and content checksums;
  (c) 256 x 4 MiB hdfs blocks with block checksums
times the three calls (one warm-up, then two alternating passes; host clock around calls that end in a device
synchronise).  A separate profiled call per frame gives the device time of the compress, block-checksum and
content-hash kernels (torch.profiler), and the content-hash rate.  Finally one profiled device call on a 64 MiB frame
with every check lists every host<->device copy, to show that nothing but the 8-byte frame length crosses PCIe."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from frame_device_probe import card, timed  # noqa: E402
from lz4_flex_b200 import _native, block, corpus, frame  # noqa: E402
from lz4_flex_b200.frame import BlockSize, FrameInfo  # noqa: E402

KERNELS = ("lz4_compress_blocks", "frame_block_checksum_kernel", "frame_batch_content_kernel", "gather_segments_kernel",
           "frame_batch_tail_kernel")


def kernel_times(fn, trace_path=None):
    """Device time per kernel family (ms) and the host<->device copies of one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    path = trace_path or os.path.join(tempfile.gettempdir(), "frame_compress_device_probe.trace.json")
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
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_compress_device_probe"),
                    help="directory for the profiler trace of the 64 MiB frame")
    ap.add_argument("--gib", type=float, default=1.0)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    print("card:", card(), flush=True)
    L = _native.lib()
    ctx = block.Context(0)
    s = torch.cuda.current_stream().cuda_stream
    total = int(args.gib * (1 << 30))
    json_data = corpus.tiled("compression_66k_JSON.txt", total)
    hdfs = corpus.tiled("hdfs.json", 256 << 22)
    cases = [
        ("a: 64 KiB JSON blocks, no checksums", json_data, FrameInfo(block_size=BlockSize.Max64KB)),
        ("b: 64 KiB JSON blocks, block + content checksums", json_data,
         FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True)),
        ("c: 256 x 4 MiB hdfs blocks, block checksums", hdfs,
         FrameInfo(block_size=BlockSize.Max4MB, block_checksums=True)),
    ]
    rows = []
    for name, data, info in cases:
        ci = info.to_c()
        n = data.size
        bsz = info.block_size.get_size()
        cap = L.lz4b200_frame_bound(n, C.byref(ci))
        h_in = torch.from_numpy(data).pin_memory()
        h_out = torch.empty(cap, dtype=torch.uint8).pin_memory()
        d_in = h_in.cuda()
        d_out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        d_floor = torch.empty(L.lz4b200_frame_blocks_bound(n, bsz), dtype=torch.uint8, device="cuda")
        d_total = torch.empty(1, dtype=torch.int64, device="cuda")
        hw = C.c_size_t(0)
        got = {}

        def dev():
            got["dev"] = frame.compress_frame_device(d_in, info, out=d_out, ctx=ctx)

        def host():
            assert L.lz4b200_frame_compress(ctx.handle, h_in.data_ptr(), n, C.byref(ci), n, h_out.data_ptr(), cap,
                                            C.byref(hw)) == 0

        def floor():
            assert L.lz4b200_frame_compress_blocks_device(ctx.handle, d_in.data_ptr(), n, bsz, 0, d_floor.data_ptr(),
                                                          d_floor.numel(), d_total.data_ptr(), None, s) == 0

        dev(); host(); floor()                                                   # warm-up, and the outputs checked
        torch.cuda.synchronize()
        assert got["dev"].numel() == hw.value, name
        assert torch.equal(got["dev"].cpu(), h_out[:hw.value]), name
        t = {"device": [], "floor": [], "host": []}
        for _ in range(2):
            t["device"].append(timed(dev)); t["floor"].append(timed(floor)); t["host"].append(timed(host))
        k, _ = kernel_times(dev)
        hash_ms = k["frame_batch_content_kernel"][1]
        row = {"frame": name, "input_bytes": int(n), "frame_bytes": hw.value, "blocks": (n + bsz - 1) // bsz,
               "ms": {m: [round(v, 2) for v in vs] for m, vs in t.items()},
               "kernels_ms": {m: {"launches": c, "ms": round(ms, 3)} for m, (c, ms) in k.items()},
               "content_hash_GBps": round(n / hash_ms / 1e6, 3) if hash_ms else None}
        rows.append(row)
        print(json.dumps(row), flush=True)
        del d_in, d_out, d_floor, h_in, h_out, got
        torch.cuda.empty_cache()

    # ---- nothing but the frame length crosses PCIe: every copy of one device call on 64 MiB with every check ------------
    data = corpus.tiled("compression_66k_JSON.txt", 64 << 20)
    info = FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True, content_size=data.size)
    d_in = torch.from_numpy(data).cuda()
    want = frame.compress_frame(data, info, ctx)
    frame.compress_frame_device(d_in, info, ctx=ctx)
    got = {}
    k, copies = kernel_times(lambda: got.setdefault("f", frame.compress_frame_device(d_in, info, ctx=ctx)),
                             os.path.join(args.out, "frame_compress_device_64mib.pt.trace.json"))
    assert got["f"].cpu().numpy().tobytes() == want
    summary = {}
    for m, b in copies:
        e = summary.setdefault(m, {"count": 0, "bytes": 0, "largest": 0})
        e["count"] += 1; e["bytes"] += b; e["largest"] = max(e["largest"], b)
    print(json.dumps({"trace_64mib": {"frame_bytes": len(want), "copies": summary,
                                      "kernels_ms": {m: {"launches": c, "ms": round(ms, 3)} for m, (c, ms) in k.items()}}}),
          flush=True)
    largest = max((b for _, b in copies), default=0)
    assert largest <= 8, f"a copy of {largest} bytes crossed PCIe"
    print("ok")


if __name__ == "__main__":
    main()
