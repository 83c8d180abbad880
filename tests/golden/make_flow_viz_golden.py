"""Regenerate tests/golden/flow_viz.npz: the reference's own `flow_to_image` on the seeded flows of
`oracle.flow_viz_np.golden_cases()`.

    python tests/golden/make_flow_viz_golden.py --reference /path/to/tf-raft

The reference's tf_raft/datasets/flow_viz.py is imported from the given checkout when this runs (it needs NumPy only);
nothing of it is copied.  Only the uint8 outputs are stored; the tests regenerate the inputs from the seeds.  The result
depends on the NumPy build's float32 arctan2 (see DESIGN.md section 3.5): it was made with NumPy 2.3.5 on an x86 host
with AVX-512.
"""
import argparse
import importlib.util
import os
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), '..', '..'))
sys.path.insert(0, ROOT)

from oracle import flow_viz_np  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'flow_viz.npz')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reference', required=True, help='checkout of tf-raft (the directory holding tf_raft/)')
    args = ap.parse_args()
    path = os.path.join(args.reference, 'tf_raft', 'datasets', 'flow_viz.py')
    spec = importlib.util.spec_from_file_location('reference_flow_viz', path)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    out = {}
    with np.errstate(over='ignore', invalid='ignore'):
        for name, (flow, kw) in flow_viz_np.golden_cases().items():
            out[name] = ref.flow_to_image(flow, **kw)
    out['numpy_version'] = np.array(np.__version__)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT))


if __name__ == '__main__':
    main()
