"""Development aid: the batch frame decoder (lz4b200_frame_decompress_batch_device) against the one-frame device call
(lz4b200_frame_decompress_next_device) in a loop and the block-batch floor (lz4b200_decompress_batch_device).

    python tests/dev/frame_batch_device_probe.py [--out DIR]

Prints the card and its power limit, checks every output against the input, then for
  (a) 16 384 single-block frames of 64 KiB JSON (1 GiB decoded), no checksums: the batch call at the default frame
      budget and at a budget that holds the whole batch in one group, the block-batch floor on the same raw blocks,
      and the one-frame loop over the first 512 frames (reported per frame);
  (b) the same frames with block and content checksums;
  (c) 256 copies of tests/golden/linked/json_1m_256k_linked.lz4 in one call, and the one-frame loop over them
times each call (one warm-up, then two alternating passes; host clock around calls that end in a device
synchronise).  A separate profiled batch call per case gives the device time of each kernel (torch.profiler)."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402
from lz4_flex_b200 import _native, block, corpus  # noqa: E402

N, BS = 16384, 65536


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else torch.cuda.get_device_name(0)


def i64(v):
    return torch.tensor(np.asarray(v, dtype=np.int64), device="cuda")


class Case:
    def __init__(self, frames, out_sizes):
        self.n = len(frames)
        lens = np.array([len(f) for f in frames], dtype=np.int64)
        self.off = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.int64)
        self.d_in = torch.from_numpy(np.frombuffer(b"".join(frames), dtype=np.uint8).copy()).cuda()
        caps = np.array(out_sizes, dtype=np.int64)
        self.ooff = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
        self.d_off, self.d_len, self.d_ooff, self.d_ocap = i64(self.off), i64(lens), i64(self.ooff), i64(caps)
        self.lens, self.caps = lens, caps
        self.d_out = torch.empty(int(caps.sum()), dtype=torch.uint8, device="cuda")
        self.res = torch.zeros((self.n, 5), dtype=torch.int64, device="cuda")

    def batch(self, ctx):
        s = torch.cuda.current_stream().cuda_stream
        st = _native.lib().lz4b200_frame_decompress_batch_device(
            ctx.handle, self.d_in.data_ptr(), self.d_off.data_ptr(), self.d_len.data_ptr(), self.d_out.data_ptr(),
            self.d_ooff.data_ptr(), self.d_ocap.data_ptr(), self.res.data_ptr(), self.n, s)
        assert st == 0, ctx.last_cuda_error()

    def loop(self, ctx, count):
        s = torch.cuda.current_stream().cuda_stream
        base_in, base_out = self.d_in.data_ptr(), self.d_out.data_ptr()
        used, w, bs, e1, e2 = C.c_size_t(0), C.c_size_t(0), C.c_int(0), C.c_uint64(0), C.c_uint64(0)
        for i in range(count):
            st = _native.lib().lz4b200_frame_decompress_next_device(
                ctx.handle, base_in + int(self.off[i]), int(self.lens[i]), base_out + int(self.ooff[i]),
                int(self.caps[i]), C.byref(used), C.byref(w), C.byref(bs), C.byref(e1), C.byref(e2), s)
            assert st == 0, st


def timed(fn, reps=1):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def kernel_times(fn, trace):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    prof.export_chrome_trace(trace)
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
        if t and "Memcpy" not in e.key and "Memset" not in e.key and "cuda" not in e.key[:4]:
            out[e.key.split("(")[0][:60]] = round(t / 1e3, 3)
    return dict(sorted(out.items(), key=lambda kv: -kv[1])[:10])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "frame_batch_device_probe"))
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    print("card:", card())
    ctx, whole = block.Context(0), block.Context(0)
    _native.lib().lz4b200_ctx_set_frame_budget(whole.handle, 4 << 30)
    data = corpus.tiled("compression_66k_JSON.txt", N * BS)
    raw = [data[i * BS:(i + 1) * BS].tobytes() for i in range(N)]
    plain = Case([oracle.frame_compress(r, 4, 0) for r in raw], [BS] * N)
    checked = Case([oracle.frame_compress(r, 4, oracle.F_BLOCK_CHECKSUMS | oracle.F_CONTENT_CHECKSUM) for r in raw],
                   [BS] * N)
    lk = open(os.path.join(ROOT, "tests", "golden", "linked", "json_1m_256k_linked.lz4"), "rb").read()
    lk_raw = oracle.frame_decompress(lk, 4 << 20)[1]
    linked = Case([lk] * 256, [len(lk_raw)] * 256)

    # the floor: the same raw blocks (payload after the 7-byte header and the 4-byte BlockInfo) as a block batch
    f_off = torch.from_numpy(plain.off + 11).cuda()
    f_len = (plain.d_len - 15).to(torch.int32)
    f_oo = torch.arange(N, dtype=torch.int64, device="cuda") * BS
    f_cap = torch.full((N,), BS, dtype=torch.int32, device="cuda")
    f_ol = torch.zeros(N, dtype=torch.int32, device="cuda")
    f_st = torch.zeros(N, dtype=torch.int32, device="cuda")

    def floor():
        st = _native.lib().lz4b200_decompress_batch_device(
            ctx.handle, plain.d_in.data_ptr(), f_off.data_ptr(), f_len.data_ptr(), plain.d_out.data_ptr(),
            f_oo.data_ptr(), f_cap.data_ptr(), f_ol.data_ptr(), f_st.data_ptr(), None, N, torch.cuda.current_stream().cuda_stream)
        assert st == 0

    want = torch.from_numpy(data).cuda()
    for c in (plain, checked):
        for x in (ctx, whole):
            c.d_out.zero_()
            c.batch(x)
            r = c.res.cpu().numpy()
            assert (r[:, 4] == 0).all() and (r[:, 1] == BS).all() and torch.equal(c.d_out, want)
    floor()
    assert not f_st.any() and torch.equal(plain.d_out, want)
    linked.batch(ctx)
    assert (linked.res.cpu().numpy()[:, 4] == 0).all()
    assert linked.d_out[:len(lk_raw)].cpu().numpy().tobytes() == lk_raw
    print("outputs verified")

    rows = {}
    runs = [("a batch, default budget", lambda: plain.batch(ctx)), ("a batch, one group", lambda: plain.batch(whole)),
            ("a decompress_batch_device floor", floor),
            ("a one-frame loop, per frame (512)", lambda: plain.loop(ctx, 512)),
            ("b batch, default budget", lambda: checked.batch(ctx)), ("b batch, one group", lambda: checked.batch(whole)),
            ("b one-frame loop, per frame (512)", lambda: checked.loop(ctx, 512)),
            ("c batch, 256 linked frames", lambda: linked.batch(ctx)),
            ("c one-frame loop, 256 frames", lambda: linked.loop(ctx, 256))]
    for _, fn in runs:
        fn()
    for p in range(2):
        for name, fn in runs:
            t = timed(fn)
            if "per frame" in name:
                t /= 512
            rows.setdefault(name, []).append(round(t, 4))
    for name, ts in rows.items():
        print(f"{name:40s} {ts} ms")
    kt = {}
    for name, fn in (("a_default", lambda: plain.batch(ctx)), ("a_one_group", lambda: plain.batch(whole)),
                     ("b_default", lambda: checked.batch(ctx)), ("c_linked", lambda: linked.batch(ctx))):
        kt[name] = kernel_times(fn, os.path.join(args.out, f"{name}.pt.trace.json"))
        print(name, json.dumps(kt[name]))
    with open(os.path.join(args.out, "frame_batch_device_probe.json"), "w") as fh:
        json.dump({"card": card(), "times_ms": rows, "kernels_ms": kt}, fh, indent=1)
    ctx.close()
    whole.close()


if __name__ == "__main__":
    main()
