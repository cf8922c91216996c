"""Compares the real crate's linked frames (written by `cargo run --release -- <benches> <out>`) with the linked-frame
reference's frames (tests/cpp/linked_frame_ref.c) of the same corpus, block size and flags:
    python compare.py <out>
Exit 0 means every frame is byte-identical, which pins the reference, and through it the GPU encoder, to the crate."""
import os
import sys

here = os.path.dirname(os.path.abspath(__file__))
root = os.path.dirname(os.path.dirname(os.path.dirname(here)))
sys.path.insert(0, root)
sys.path.insert(0, os.path.join(root, "tests"))
import linked_ref  # noqa: E402
from lz4_flex_b200 import corpus  # noqa: E402

out = sys.argv[1]
ok = bad = 0
for fn in sorted(os.listdir(out)):
    if not fn.endswith(".frame.lz4") or ".linked_" not in fn:
        continue
    name, spec = fn[:-len(".frame.lz4")].split(".linked_")
    bsid, flags = (int(x) for x in spec.split("_"))
    good = open(os.path.join(out, fn), "rb").read() == linked_ref.frame_compress(corpus.load(name), bsid, flags)
    ok += good
    bad += not good
    if not good:
        print("MISMATCH", fn)
print(f"{ok} match, {bad} mismatch")
sys.exit(1 if bad or not ok else 0)
