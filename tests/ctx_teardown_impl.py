"""Child process of tests/test_gpu_ctx_teardown.py.

One context runs each kind of call that reserves scratch once, on inputs of a few MiB: the host block batch with and
without a dictionary, the host frame calls on an independent-block frame and on a linked frame, the device batch frame
encoder and decoder, the size-prepended device batch, and a streaming decoder and encoder.  Then the context is
destroyed and every tensor is released.  This runs twice, each time on a new context.  The first pass lets torch create
what it keeps for the whole process (its stream pool and pinned staging); the second runs under torch.profiler, which
records every CUDA runtime call of the process.  With torch's caching allocator off (PYTORCH_NO_CUDA_MEMORY_CACHING=1)
each tensor frees its own device memory.  The last line printed is a JSON object with the number of each CUDA runtime
call of the second pass."""
import gc
import hashlib
import json
import os
import re
import sys
from collections import Counter

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from lz4_flex_b200 import block, corpus, frame  # noqa: E402
from lz4_flex_b200.frame import BlockSize, FrameInfo  # noqa: E402

KiB, MiB = 1 << 10, 1 << 20


def workload(dev, data):
    ctx = block.Context(0)
    blocks = [data[i:i + 64 * KiB] for i in range(0, len(data), 64 * KiB)]
    caps = [64 * KiB] * len(blocks)

    comp = block.compress_blocks(blocks, ctx=ctx)
    outs, status, _ = block.decompress_blocks(comp, caps, ctx=ctx)
    assert not status.any() and outs == blocks
    ext = data[:32 * KiB]
    comp = block.compress_blocks_with_dict(blocks, ext, ctx=ctx)
    outs, status, _ = block.decompress_blocks_with_dict(comp, caps, ext, ctx=ctx)
    assert not status.any() and outs == blocks

    info = FrameInfo(block_size=BlockSize.Max64KB, block_checksums=True, content_checksum=True)
    f = frame.compress_frame(data, info, ctx=ctx)
    out, used, err = frame.decompress_next_frame(f, ctx=ctx)
    assert err is None and used == len(f) and out == data
    gdir = os.path.join(ROOT, "tests", "golden", "linked")
    entry = next(e for e in json.load(open(os.path.join(gdir, "manifest.json"))) if e["source"] == "json_1m")
    linked = open(os.path.join(gdir, entry["file"]), "rb").read()
    out, used, err = frame.decompress_next_frame(linked, ctx=ctx)
    assert err is None and used == len(linked) and hashlib.sha256(out).hexdigest() == entry["source_sha256"]

    d_in = torch.frombuffer(bytearray(data), dtype=torch.uint8).to(dev)
    offs, lens = [0, 1 * MiB, 1 * MiB + 4096], [1 * MiB, 4096, 1 * MiB - 4096]
    frames, foff = frame.compress_frames_device(d_in, offs, lens, info, ctx=ctx)
    fo = foff.cpu().tolist()
    decoded = frame.decompress_frames_device(frames, fo[:-1], [b - a for a, b in zip(fo, fo[1:])], ctx=ctx)
    for i, (o, n) in enumerate(zip(offs, lens)):
        got, _, err = decoded.frame(i)
        assert err is None and bytes(got.cpu().numpy()) == data[o:o + n]

    recs, rec_off, rstat = block.compress_prepend_size_device(d_in, offs, lens, ctx=ctx)
    ro = rec_off.cpu().tolist()
    plain, _, _, pstat, _ = block.decompress_size_prepended_device(recs, ro[:-1], [b - a for a, b in zip(ro, ro[1:])],
                                                                   ctx=ctx)
    torch.cuda.synchronize()
    assert not rstat.any() and not pstat.any() and bytes(plain.cpu().numpy()) == data

    enc = frame.DeviceFrameEncoder(info, ctx=ctx)
    stream_frame = enc.write(d_in, finish=True)
    enc.close()
    dec = frame.DeviceFrameDecoder(ctx=ctx)
    d_out = torch.empty(len(data), dtype=torch.uint8, device=dev)
    consumed, written, _, done, err = dec.decode(stream_frame, d_out, end_of_input=True)
    dec.close()
    assert err is None and done and consumed == stream_frame.numel() and written == len(data)
    assert bytes(d_out.cpu().numpy()) == data
    ctx.close()


def main():
    assert os.environ.get("PYTORCH_NO_CUDA_MEMORY_CACHING") == "1"
    dev = torch.device("cuda", 0)
    data = corpus.tiled("compression_66k_JSON.txt", 2 * MiB).tobytes()
    workload(dev, data)
    gc.collect()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        workload(dev, data)
        gc.collect()
        torch.cuda.synchronize()
    calls = Counter(re.sub(r"_v\d+$", "", e.name) for e in prof.events() if e.name.startswith("cuda"))
    print(json.dumps(dict(calls)))


if __name__ == "__main__":
    main()
