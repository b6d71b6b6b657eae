"""Runs tests/test_gpu_dense64.py::engine_cases() in a fresh process, so that an engine switch read once per process
(GPK_FP64_SIMT=1: the fp64 CUDA-core GEMM) takes effect.  Every case runs through the same assertions and bars as in
the test module; the failures and the worst error / bar of each operator are written as JSON.
Usage: python -m tests._dense64_worker OUT.json"""
import json
import os
import sys
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main(out):
    import torch

    from tests import test_gpu_dense64 as T

    torch.cuda.set_device(0)
    cases = T.engine_cases()
    failed = []
    for fn, args in cases:
        try:
            fn(None, *args)
        except AssertionError:
            failed.append(f"{fn.__name__}{args}: {traceback.format_exc(limit=1).strip().splitlines()[-1]}")
    torch.cuda.synchronize()
    with open(out, "w") as f:
        json.dump({"cases": len(cases), "failed": failed,
                   "worst": {k: [float(a), float(b)] for k, (a, b) in T.WORST.items()}}, f)


if __name__ == "__main__":
    main(sys.argv[1])
