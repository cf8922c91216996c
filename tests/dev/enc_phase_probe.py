"""Development aid (run on a GPU): the block encoder's matcher cycles per sequence, phase by phase.

Builds the library with -DLZ4B200_ENC_PROFILE into a temporary directory (or loads the library given with --so), compresses
the bench.py workload (16 384 x 64 KiB JSON blocks) once to warm up and once measured, and prints clock64() cycles per
sequence for each phase of match_block_view (summed over all matcher warps, divided by the sequences they produced), plus
the sequence statistics the extension paths depend on.  The profile build adds clock reads and registers to the matcher,
so its absolute times are not the product's; the split between phases is what it is for.

    python tests/dev/enc_phase_probe.py [--so PATH | -D MACRO=VALUE ...] [--blocks N] [--json OUT]
"""
import argparse
import json
import os
import shutil
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

PHASES = ["probe", "resolve", "commit", "extend", "push", "setup"]
COUNTS = ["sequences", "batches", "no_backward", "short_forward", "long_forward", "blocks"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--so", help="a library already built with -DLZ4B200_ENC_PROFILE")
    ap.add_argument("--blocks", type=int, default=16384)
    ap.add_argument("--json", help="also write the table to this file")
    ap.add_argument("-D", dest="defines", action="append", default=[], help="extra -D for the profile build, e.g. ENC_RI_PATCH=1")
    args = ap.parse_args()
    tmp = tempfile.mkdtemp(prefix="lz4b200_encprof_")
    try:
        so = os.path.abspath(args.so) if args.so else os.path.join(tmp, "liblz4b200_encprof.so")
        os.environ["LZ4B200_SO_OVERRIDE"] = so          # read when lz4_flex_b200._native is imported
        from lz4_flex_b200 import _native
        if not args.so:
            _native._compile(so, ["-DLZ4B200_ENC_PROFILE"] + ["-D" + d for d in args.defines], force=True)
        run(args)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def run(args):

    import ctypes as C
    import numpy as np
    import torch
    import bench
    from lz4_flex_b200 import _native, block

    L = _native.lib()
    L.lz4b200_enc_profile_read.restype = C.c_int
    L.lz4b200_enc_profile_read.argtypes = [C.POINTER(C.c_uint64), C.c_int]
    nb, B, slot = args.blocks, bench.BLOCK, 72112
    dev = torch.device("cuda", 0)
    ctx = block.Context(0)
    data = bench.build_workload(nb, 0)
    d_in = torch.from_numpy(data).to(dev)
    d_comp = torch.zeros(nb * slot, dtype=torch.uint8, device=dev)
    enc = block.DeviceBatch(np.arange(nb, dtype=np.uint64) * B, np.full(nb, B, dtype=np.uint32),
                            np.arange(nb, dtype=np.uint64) * slot, np.full(nb, slot, dtype=np.uint32), None, dev)
    buf = (C.c_uint64 * 16)()
    enc.compress(d_in, d_comp, ctx)
    assert L.lz4b200_enc_profile_read(buf, 1) == 0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    enc.compress(d_in, d_comp, ctx)
    e1.record()
    assert L.lz4b200_enc_profile_read(buf, 1) == 0
    assert int(enc.status.abs().sum()) == 0
    kernel = _native.lib().lz4b200_ctx_last_kernel(ctx.handle, 0).decode()
    v = list(buf)
    seqs = max(v[6], 1)
    phases = {name: v[i] / seqs for i, name in enumerate(PHASES)}
    counts = {name: v[6 + i] for i, name in enumerate(COUNTS)}
    rec = {"kernel": kernel, "blocks": nb, "compress_ms_profile_build": e0.elapsed_time(e1),
           "device": torch.cuda.get_device_name(0), "cycles_per_sequence": phases,
           "cycles_per_sequence_total": sum(phases.values()), "counts": counts,
           "batches_per_sequence": v[7] / seqs, "sequences_per_block": v[6] / max(v[11], 1),
           "no_backward_frac": v[8] / seqs, "short_forward_frac": v[9] / seqs, "long_forward_frac": v[10] / seqs}
    print(f"{kernel}: {nb} blocks, {v[6]} sequences ({rec['sequences_per_block']:.0f} per block), "
          f"{rec['batches_per_sequence']:.3f} probe batches per sequence; profile build {rec['compress_ms_profile_build']:.2f} ms")
    for name in PHASES:
        print(f"  {name:8s} {phases[name]:9.1f} cycles/sequence  {100 * phases[name] / rec['cycles_per_sequence_total']:5.1f} %")
    print(f"  {'total':8s} {rec['cycles_per_sequence_total']:9.1f}")
    print(f"  no backward round {100 * rec['no_backward_frac']:.1f} %, of all sequences ending within 8 bytes without one "
          f"{100 * rec['short_forward_frac']:.1f} %, longer than 36 bytes {100 * rec['long_forward_frac']:.1f} %")
    print(json.dumps(rec))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
