"""Run the REFERENCE's INT4 quantise / dequantise kernels (demo/quantize_int4.cu, built into oracle/_ref/ by
oracle/build_ref.py with the reference's own --use_fast_math) on a GPU and store their outputs in
int4_reference_kernels.npz, the fixture of tests/test_gpu_kv_ops.py::test_quant_dequant_vs_reference_kernels_compiled_from_source.

    python tests/golden/make_golden_int4_kernels.py      (needs a CUDA device and a built oracle/_ref)

The input is regenerated from its seed by ``int4_kernel_input`` (shared with the test); the fixture keeps every
packed code and scale / zero, and a seeded sample of the dequantised rows (the whole output would pass 1 MB).
"""
from __future__ import annotations

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
FIXTURE = os.path.join(HERE, "int4_reference_kernels.npz")
SHAPE = (2, 300, 4)  # (batch, tokens, heads) of 128-element groups
N_DEQUANT_SAMPLE = 256


def int4_kernel_input():
    rng = np.random.RandomState(2)
    return (rng.randn(*SHAPE, 128) * rng.uniform(0.05, 5, size=(*SHAPE, 1))).astype(np.float16)


def dequant_sample_rows():
    return np.sort(np.random.RandomState(3).choice(int(np.prod(SHAPE)), N_DEQUANT_SAMPLE, replace=False))


def main():
    import torch

    sys.path.insert(0, ROOT)
    from oracle import build_ref

    ref = build_ref.load_module()
    if ref is None:
        raise SystemExit("oracle/_ref is not built (oracle/build_ref.py needs the reference sources)")
    dev = torch.device("cuda")
    x = int4_kernel_input()
    rows = int(np.prod(SHAPE))
    xt = torch.from_numpy(x).to(dev)
    qp = torch.empty(*SHAPE, 64, dtype=torch.uint8, device=dev)
    sc = torch.empty(*SHAPE, 1, dtype=torch.float16, device=dev)
    zp = torch.empty(*SHAPE, 1, dtype=torch.float16, device=dev)
    ref.quantize_int4_with_zero_point_per_group(xt, qp, sc, zp, 128)
    buf = torch.empty(rows * 128, dtype=torch.float16, device=dev)
    ref.dequantize_int4_with_zero_point_per_group(qp.view(-1, 64), sc, zp, 128, buf, rows)
    torch.cuda.synchronize()
    sample = dequant_sample_rows()
    np.savez_compressed(FIXTURE, packed=qp.cpu().numpy().reshape(rows, 64), scale=sc.cpu().numpy().reshape(rows),
                        zero=zp.cpu().numpy().reshape(rows), dequant_rows=sample,
                        dequant=buf.cpu().numpy().reshape(rows, 128)[sample],
                        input_checksum=np.float64(x.astype(np.float64).sum()))
    print("wrote", FIXTURE, os.path.getsize(FIXTURE), "bytes")


if __name__ == "__main__":
    main()
