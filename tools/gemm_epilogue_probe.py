#!/usr/bin/env python
"""How much of the correlation GEMM's time its epilogue takes, on bench.py's headline step.

    python tools/gemm_epilogue_probe.py [rounds]

Runs the symmetric pipeline over all rows at V = 50 000, T = 200, E = 32, fp16x3 (bench.py's inputs, workspace and
passes) with the diagnostic build's knobs, the variants alternating in one process:
  full      the product kernel;
  no-store  the epilogue math with its result kept live but no store issued (FCMA_GEMM_EPILOGUE=1);
  none      no epilogue (FCMA_GEMM_EPILOGUE=2).
Prints the GEMM time per step (CUDA events around every GEMM launch, summed over the step's passes) of each variant
and round, and the card's name and power limit.  Only `full` computes valid kernels."""
import ctypes
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import bench  # noqa: E402
from brainiak_b200 import _lib  # noqa: E402
from brainiak_b200 import build as _build  # noqa: E402

_build.build(diag=True)
_lib.use_diag_build()
from brainiak_b200.fcma import engine  # noqa: E402

VARIANTS = (("full", "0"), ("no-store", "1"), ("none", "2"))


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    lib = _lib.load()
    dev = torch.device("cuda:0")
    V, T, E, eps = (bench.WORKLOAD[k] for k in ("V", "T", "E", "eps"))
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("device: %s | nvidia-smi: %s" % (torch.cuda.get_device_name(dev), smi), flush=True)
    epochs = bench.make_host_epochs(V, T, E).to(dev)
    op = engine.pack_epochs(epochs, None, "fp16x3")
    code = _lib.PREC["fp16x3"]
    cols = bool(lib.fcma_sym_uses_column_pass(code, E, eps, 0))
    work = engine.SymWorkspace(E, V, 4096, dev, start=0, transposed_copy=not cols)
    K = torch.zeros((V, E, E), device=dev)

    def step():
        K.zero_()
        engine.voxel_kernels_sym(op, 0, V, eps, flags=0, work=work, out=K)

    times = {name: [] for name, _ in VARIANTS}
    for r in range(rounds):
        for name, knob in VARIANTS:
            os.environ["FCMA_GEMM_EPILOGUE"] = knob
            step()                      # warm-up of this variant's kernel
            torch.cuda.synchronize()
            lib.fcma_timing_enable(1)
            step()
            step()
            torch.cuda.synchronize()
            g = ctypes.c_double(0)
            npass = lib.fcma_timing_read3(ctypes.byref(g), None, None)
            lib.fcma_timing_enable(0)
            times[name].append(g.value / 2)
            print("round %d  %-8s  GEMM %.2f ms per step (%d passes)" % (r, name, g.value / 2, npass // 2), flush=True)
    os.environ.pop("FCMA_GEMM_EPILOGUE", None)
    for name, _ in VARIANTS:
        t = sorted(times[name])
        print("%-8s  GEMM ms per step: min %.2f  median %.2f  max %.2f" % (name, t[0], t[len(t) // 2], t[-1]))


if __name__ == "__main__":
    main()
