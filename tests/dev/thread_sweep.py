"""Dev sweep (on a GPU): K1-T / K2-T launch shapes vs the warp-cooperative kernels on config 2 (and 3).
Usage: python tests/dev/thread_sweep.py [nblocks] ; prints one line per shape: compress ms, decompress ms, parity."""
import hashlib, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import numpy as np
import torch
import oracle
from lz4_flex_b200 import _native
if "LZ4B200_SO_OVERRIDE" not in os.environ:                  # the A/B library carries every variant and its switches
    os.environ["LZ4B200_SO_OVERRIDE"] = _native.build_ab()
    os.execv(sys.executable, [sys.executable] + sys.argv)
from lz4_flex_b200 import block, corpus

NB = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
FILE = sys.argv[2] if len(sys.argv) > 2 else "compression_66k_JSON.txt"
BS = 65536
dev = torch.device("cuda", 0)
data = corpus.tiled(FILE, NB * BS)
stride = (block.get_maximum_output_size(BS) + 15) // 16 * 16
in_off = np.arange(NB, dtype=np.uint64) * BS
in_len = np.full(NB, BS, dtype=np.uint32)
out_off = np.arange(NB, dtype=np.uint64) * stride
out_cap = np.full(NB, stride, dtype=np.uint32)
# oracle reference (all blocks)
t0 = time.time()
ref = np.zeros(NB * stride, dtype=np.uint8)
ref_len, ref_st = oracle.compress_batch(data, in_off, in_len, ref, out_off, out_cap, os.cpu_count())
print(f"oracle compress of {NB} blocks: {time.time() - t0:.2f}s, ratio {ref_len.sum() / data.size:.4f}", flush=True)
def packed_sha(buf, lens):
    h = hashlib.sha256()
    for b in range(NB):
        h.update(buf[b * stride:b * stride + int(lens[b])].tobytes())
    return h.hexdigest()
ref_sha = packed_sha(ref, ref_len)

d_in = torch.from_numpy(data).to(dev)
d_comp = torch.zeros(NB * stride, dtype=torch.uint8, device=dev)
d_back = torch.zeros(NB * BS, dtype=torch.uint8, device=dev)

def run(env, label, iters=5):
    for k in list(os.environ):
        if k.startswith("LZ4B200_") and k != "LZ4B200_SO_OVERRIDE":
            del os.environ[k]
    os.environ.update(env)
    ctx = block.Context(0)
    cb = block.DeviceBatch(in_off, in_len, out_off, out_cap)
    d_comp.zero_(); d_back.zero_()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    cms, dms = [], []
    db = None
    for it in range(iters):
        torch.cuda.synchronize()
        ev[0].record(); cb.compress(d_in, d_comp, ctx); ev[1].record()
        torch.cuda.synchronize()
        if db is None:
            clen = cb.out_len.cpu().numpy().astype(np.uint32)
            assert (cb.status.cpu().numpy() == 0).all()
            db = block.DeviceBatch(out_off, clen, in_off, in_len)
        ev[2].record(); db.decompress(d_comp, d_back, ctx); ev[3].record()
        torch.cuda.synchronize()
        cms.append(ev[0].elapsed_time(ev[1])); dms.append(ev[2].elapsed_time(ev[3]))
    comp = d_comp.cpu().numpy()
    ok_c = (clen == ref_len).all() and packed_sha(comp, clen) == ref_sha
    ok_d = bool((d_back == d_in).all().item()) and (db.status.cpu().numpy() == 0).all() and (db.out_len.cpu().numpy() == BS).all()
    print(f"{label:44s} compress {min(cms[1:]):8.3f} ms  decompress {min(dms[1:]):8.3f} ms  parity c={ok_c} d={ok_d}", flush=True)
    ctx.close()

MODE = sys.argv[3] if len(sys.argv) > 3 else "gtag"
if MODE == "plain":
    run({}, "default launch policy of " + os.path.basename(os.environ["LZ4B200_SO_OVERRIDE"]))
elif MODE == "thread":
    run({"LZ4B200_THREAD_MIN": "4000000000"}, "round-1 warp kernels (gtab / G=8)")
    for lanes in (32, 16, 8):
        run({"LZ4B200_THREAD_MIN": "1", "LZ4B200_ENC_THREAD_LANES": str(lanes), "LZ4B200_DEC_THREAD_LANES": str(lanes)}, f"thread kernels, {lanes} lanes/warp")
elif MODE == "nib":
    run({}, "gtab 7+1 x8 (default)")
    for mode, ctas, what in (("2", 6, "byte tags, 32 lanes"), ("4", 4, "2-bit tags, 8-lane groups"), ("4", 3, "2-bit tags, 8-lane groups"),
                             ("5", 8, "2-bit tags, 16-lane groups"), ("5", 6, "2-bit tags, 16-lane groups")):
        run({"LZ4B200_ENC_NIB": mode, "LZ4B200_ENC_NIB_CTAS": str(ctas)}, f"smem {what}, first-2 verify, {ctas} CTAs/SM", iters=4)
elif MODE == "g16":
    run({}, "gtab 7+1 x8 (round 1 default)")
    for shape, ctas_list in (("71", (8, 4)), ("871", (8, 4, 2)), ("862", (8,))):
        for ctas in ctas_list:
            run({"LZ4B200_ENC_G16": shape, "LZ4B200_ENC_G16_CTAS": str(ctas)}, f"lane-group matchers {shape}, {ctas} CTAs/SM", iters=4)
else:
    run({"LZ4B200_ENC_GTAG": "0"}, "untagged gtab 7+1 x8 (round 1)")
    for ctas in (8, 7, 6, 5):
        run({"LZ4B200_ENC_GTAG": "71", "LZ4B200_ENC_GTAG_CTAS": str(ctas)}, f"tagged tables 7+1, {ctas} CTAs/SM")
    run({}, "default")
