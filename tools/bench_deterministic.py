"""bench.py's workload in deterministic mode: ``torch.use_deterministic_algorithms(True)``.

Every backward of bevformer_b200 then takes its fixed-order kernel (fixed-point sampler grad_value, ordered
LayerNorm / bias / weight-gradient reductions), and PyTorch's own ops their deterministic forms, so two runs with the
same arguments give bit-identical outputs and gradients (compare the ``--dump-outputs`` directories of two runs).
Takes bench.py's arguments and prints its JSON line.

PyTorch's NaN fill of uninitialised memory (``torch.utils.deterministic.fill_uninitialized_memory``) is switched off:
it is a debugging aid that adds a fill kernel to every ``torch.empty`` and would be billed to this mode's step time.
Usage: python tools/bench_deterministic.py --steps 10 [bench.py arguments]
"""
from __future__ import annotations

import os
import sys

# cuBLAS picks a reproducible reduction only with a fixed workspace configuration; it must be set before cuBLAS starts
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.utils.deterministic  # noqa: E402

import bench  # noqa: E402


def main():
    torch.use_deterministic_algorithms(True)
    torch.utils.deterministic.fill_uninitialized_memory = False
    print("bench_deterministic: torch.use_deterministic_algorithms(True), CUBLAS_WORKSPACE_CONFIG="
          f"{os.environ['CUBLAS_WORKSPACE_CONFIG']}, fill_uninitialized_memory off for timing", file=sys.stderr)
    try:
        bench.main()
    except RuntimeError as e:
        if "deterministic" in str(e):
            print(f"bench_deterministic: an op on the step's path has no deterministic implementation: {e}",
                  file=sys.stderr)
        raise


if __name__ == "__main__":
    main()
