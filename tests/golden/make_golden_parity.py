"""Writes tests/golden/rasterizer-reference.npz: what tests/test_gpu_parity.py compares this repository's rasterizer with.

Every case of the test module is run through Oracle-A -- the reference extension compiled in place into
oracle/_ref by oracle/build_ref.py (part of __graft_entry__.build() where the reference sources are present) --
on a GPU, and the outputs are kept as compact records (tests/_util.py `sketch`): byte digests of the arrays the
tests compare bit for bit, norm / random projections / sampled elements /
per-block maxima of the floating-point ones.

    python tests/golden/make_golden_parity.py OUT.npz        (on the GPU; then copy OUT.npz to tests/golden/rasterizer-reference.npz)
"""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
sys.path.insert(0, TESTS)

import _util  # noqa: E402
import test_gpu_parity as tp  # noqa: E402


def main(out_path):
    dev = torch.device("cuda:0")
    ref = _util.ref_module()
    records = {}
    for case, make in tp.RUN_CASES.items():
        records[case] = tp.record_run(*tp.run_rasterizer(ref._C, make(dev), dev))
        print(f"{case}: R={records[case]['R']}", flush=True)
    records["mark-visible"] = {"visible": {"digest": _util.digest(tp.mark_visible_run(ref._C, dev))}}
    for mode in tp.API_MODES:
        color, radii, grads = tp.public_api_run(ref, mode, dev)
        rec = {"color": _util.sketch(color), "radii": {"digest": _util.digest(radii)}}
        rec.update({f"grad_{k}": _util.sketch(g) for k, g in grads.items() if g is not None})
        records[f"api-{mode}"] = rec
    _util.save_records(out_path, records)
    print(out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main(sys.argv[1])
