"""Regenerate tests/golden/datasets.npz: the reference's own dataset classes run on the synthetic tree that
tests/test_datasets.py's `make_tree` writes.

    python tests/golden/make_datasets_golden.py --reference /path/to/tf-raft

The reference's tf_raft/datasets/{frame_utils,augmentor,dataset}.py are imported from the given checkout as a
package of their own (tf_raft/__init__.py, which builds the TensorFlow model, is not run).  `tensorflow` and
`albumentations` are replaced by empty modules in sys.modules: the file lists and `__getitem__` without aug_params
use neither.  OpenCV and PIL are needed.  Nothing of the reference is copied; the file stores the lists relative to
the tree's root, the extra_info and the decoded arrays of the items in test_datasets.ITEMS.
"""
import argparse
import importlib
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, '..', '..'))
sys.path.insert(0, os.path.join(HERE, '..'))

import test_datasets as T  # noqa: E402

OUT = os.path.join(HERE, 'datasets.npz')


def load_reference(checkout):
    for name in ('tensorflow', 'albumentations'):
        sys.modules.setdefault(name, types.ModuleType(name))
    pkg = types.ModuleType('reference_datasets')
    pkg.__path__ = [os.path.join(checkout, 'tf_raft', 'datasets')]
    sys.modules['reference_datasets'] = pkg
    return importlib.import_module('reference_datasets.dataset')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reference', required=True, help='checkout of tf-raft (the directory holding tf_raft/)')
    args = ap.parse_args()
    ref = load_reference(args.reference)
    out = {}
    with tempfile.TemporaryDirectory() as root:
        T.make_tree(root)
        ds = T.configs(ref, root)
        for name, d in ds.items():
            for field, value in T.describe(d, root).items():
                out[f'{name}/{field}'] = value
        for name, key in T.ITEMS:
            item = ds[name][T.item_index(ds[name], key)]
            tag = T.item_tag(name, key)
            for k, a in enumerate(item):
                out[f'item/{tag}/{k}'] = np.array('/'.join(str(x) for x in a), dtype=str) if k == 2 and ds[name].is_test \
                    else np.asarray(a)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), len(out), 'arrays')


if __name__ == '__main__':
    main()
