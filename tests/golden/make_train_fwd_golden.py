"""Runs the training forward (ops.train_fwd) on frame 0 of the oracle scene for every case of oracle/train_fwd_golden.py
and stores what tests/test_gpu_train.py and tests/test_gpu_edge_cases.py compare it against (layout described there).

The committed golden is the retired one-kernel forward's result.  Regenerate it only with a change that alters the
training forward's numerics on purpose, and say so in that change.

Usage (needs a GPU):  python tests/golden/make_train_fwd_golden.py OUT_DIR"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import testing, train_fwd_golden as tfg  # noqa: E402


def main(out_dir):
    sc = testing.oracle_scene(0)
    scene, _ = testing.upload(sc)
    out = {}
    for case in tfg.CASES:
        rec = tfg.record(*tfg.run(scene, tfg.inputs(sc, case)))
        out.update({f"{case}/{k}": v for k, v in rec.items()})
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, os.path.basename(tfg.PATH))
    np.savez_compressed(path, **out)
    print("saved", path, os.path.getsize(path), {c: out[f"{c}/stats"].tolist() for c in tfg.CASES})


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.dirname(tfg.PATH))
