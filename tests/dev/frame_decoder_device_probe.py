"""Development aid: the streaming device frame decoder (lz4b200_frame_decoder) against the one-shot device call
(lz4b200_frame_decompress_next_device) on the same frame, and the context's device memory after each.

    python tests/dev/frame_decoder_device_probe.py [--out DIR]

Prints the card and its power limit, then for
  (a) a 1 GiB frame of independent 64 KiB JSON blocks, decoded in 16, 64 and 256 MiB input chunks into a 256 MiB
      output buffer, against the one-shot call on the whole frame into 1 GiB;
  (b) a 64 MiB linked frame of 4 MiB blocks, decoded in 16 MiB input chunks into a 16 MiB output buffer, against the
      one-shot call;
the time of each (one checked warm-up, then two alternating passes; host clock around calls that end in a device
synchronise) and lz4b200_ctx_device_bytes of a fresh context (default 256 MiB frame budget) after the run."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from lz4_flex_b200 import _native, block, corpus, frame  # noqa: E402
from lz4_flex_b200.frame import BlockSize, FrameInfo  # noqa: E402
from stream_frames import linked_frame  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def one_shot(ctx, d_in, out):
    used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
    st = _native.lib().lz4b200_frame_decompress_next_device(
        ctx.handle, d_in.data_ptr(), d_in.numel(), out.data_ptr(), out.numel(), C.byref(used), C.byref(w),
        C.byref(bs), C.byref(e1), C.byref(e2), torch.cuda.current_stream().cuda_stream)
    assert st == 0 and used.value == d_in.numel(), st
    return w.value


def streamed(ctx, dec, d_in, out, chunk, src=None):
    """Presents d_in in windows of `chunk` bytes from the first unconsumed byte; checks the output against src."""
    L = _native.lib()
    step = _native.FrameDecoderStepC()
    s = torch.cuda.current_stream().cuda_stream
    pos, off, n, calls = 0, 0, d_in.numel(), 0
    while True:
        end = min(n, pos + chunk)
        st = L.lz4b200_frame_decoder_decode_device(dec, d_in[pos:].data_ptr(), end - pos, int(end == n), out.data_ptr(),
                                                   out.numel(), C.byref(step), s)
        assert st == 0, st
        calls += 1
        if src is not None and step.written:
            assert torch.equal(out[:step.written], src[off:off + step.written])
        off += step.written
        pos += step.consumed
        if step.frame_done:
            assert step.result.status == 0 and pos == n
            return off, calls


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return 1e3 * (time.perf_counter() - t0)


def measure(name, f_host, src, bs_out, chunks, rows):
    d_in = torch.from_numpy(np.frombuffer(f_host, dtype=np.uint8).copy()).cuda()
    one_ctx = block.Context(0)
    full = torch.empty(src.numel(), dtype=torch.uint8, device="cuda")
    assert one_shot(one_ctx, d_in, full) == src.numel() and torch.equal(full, src)
    del full
    runs = {"one-shot": None}
    for c in chunks:
        runs[f"decoder, {c >> 20} MiB chunks"] = c
    ctxs, decs, outs = {}, {}, {}
    for key, c in runs.items():
        if c is None:
            continue
        ctxs[key] = block.Context(0)
        h = C.c_void_p()
        assert _native.lib().lz4b200_frame_decoder_create(ctxs[key].handle, C.byref(h)) == 0
        decs[key] = h
        outs[key] = torch.empty(bs_out, dtype=torch.uint8, device="cuda")
        n, calls = streamed(ctxs[key], h, d_in, outs[key], c, src)
        assert n == src.numel()
        rows.append({"frame": name, "run": key, "calls": calls})
    times = {k: [] for k in runs}
    for _ in range(2):
        for key, c in runs.items():
            if c is None:
                full = torch.empty(src.numel(), dtype=torch.uint8, device="cuda")
                times[key].append(timed(lambda: one_shot(one_ctx, d_in, full)))
                del full
            else:
                times[key].append(timed(lambda: streamed(ctxs[key], decs[key], d_in, outs[key], c)))
    for key, c in runs.items():
        cx = one_ctx if c is None else ctxs[key]
        row = {"frame": name, "run": key, "ms": [round(t, 1) for t in times[key]],
               "ctx_device_bytes": int(_native.lib().lz4b200_ctx_device_bytes(cx.handle))}
        rows.append(row)
        print(json.dumps(row), flush=True)
    for key, h in decs.items():
        _native.lib().lz4b200_frame_decoder_destroy(h)
        ctxs[key].close()
    one_ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    rows = [{"card": card()}]
    print(json.dumps(rows[0]), flush=True)
    ctx = block.default_context()

    j = corpus.tiled("compression_66k_JSON.txt", 1 << 30)
    f = frame.compress_frame(j.tobytes(), FrameInfo(block_size=BlockSize.Max64KB), ctx=ctx)
    measure("1 GiB independent 64 KiB JSON", f, torch.from_numpy(j).cuda(), 256 << 20, [16 << 20, 64 << 20, 256 << 20], rows)

    d = corpus.load("dickens.txt")
    data = (d * (1 + (64 << 20) // len(d)))[:64 << 20]
    lf = linked_frame(data, [4 << 20], 7)
    measure("64 MiB linked 4 MiB blocks", lf, torch.from_numpy(np.frombuffer(data, dtype=np.uint8).copy()).cuda(),
            16 << 20, [16 << 20], rows)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        json.dump(rows, open(os.path.join(args.out, "frame_decoder_device_probe.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
