#!/usr/bin/env python
"""Golden outputs of the reference's checkpoint / camera-file helpers (data/datasets/utils.py, numpy only) on the fixed inputs
of tests/test_checkpoint_io.py.  Run where a reference checkout exists:

    python tests/golden/make_golden_dataset_utils.py <reference root>

writes tests/golden/dataset_utils.npz (paths relative to the scratch directory the inputs were written to)."""
import importlib.util
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from test_checkpoint_io import CKPT_NAMES, camera_inputs  # noqa: E402


def main(ref_root):
    spec = importlib.util.spec_from_file_location("_ref_dataset_utils", os.path.join(ref_root, "data", "datasets", "utils.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    with tempfile.TemporaryDirectory() as d:
        empty = ref.get_iteration_path(d)
        for name in CKPT_NAMES:
            open(os.path.join(d, name), "w").close()
        latest = os.path.relpath(ref.get_iteration_path(d), d)
        fixed = os.path.relpath(ref.get_iteration_path(d, 7), d)
        Ks, poses = camera_inputs()
        fn = os.path.join(d, "K.txt")
        np.savetxt(fn, Ks)
        intr = ref.read_intrinsics(fn)
        ext = ref.campose_to_extrinsic(poses)
    np.savez_compressed(os.path.join(HERE, "dataset_utils.npz"), empty_dir_is_none=np.array(empty is None),
                        latest=np.array(latest), fix_iter_7=np.array(fixed), read_intrinsics=intr, campose_to_extrinsic=ext)


if __name__ == "__main__":
    main(sys.argv[1])
