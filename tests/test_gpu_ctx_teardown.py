"""Destroying a context frees all of its device memory, pinned memory and streams.

tests/ctx_teardown_impl.py runs every kind of call that reserves context scratch once on one context, destroys the
context and releases its tensors, all under torch.profiler, and reports how often the process called each CUDA
runtime function in that window.  Every allocation must have been freed and every stream destroyed by the end.
compute-sanitizer's leak check would name the leaked allocations, but it does not support every device this suite
runs on; the runtime's own call counts do not depend on the device."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_ctx_destroy_frees_every_allocation():
    env = dict(os.environ, PYTORCH_NO_CUDA_MEMORY_CACHING="1")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "ctx_teardown_impl.py")], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    calls = json.loads(r.stdout.strip().splitlines()[-1])
    n = lambda *names: sum(calls.get(k, 0) for k in names)  # noqa: E731
    assert n("cudaStreamCreateWithPriority") >= 8, f"the host pipeline's lanes were not traced: {calls}"
    assert n("cudaMalloc") == n("cudaFree"), calls
    assert n("cudaHostAlloc", "cudaMallocHost") == n("cudaFreeHost"), calls
    assert n("cudaStreamCreate", "cudaStreamCreateWithFlags", "cudaStreamCreateWithPriority") == n("cudaStreamDestroy"), calls
