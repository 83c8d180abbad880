"""Score a TF checkpoint of tf-raft on a dataset checkout; prints one JSON line.

    python scripts/evaluate.py sintel --root datasets/MPI-Sintel-complete --checkpoint checkpoints/model [--dstype final]
    python scripts/evaluate.py kitti --root datasets/KITTI --checkpoint checkpoints/model

Defaults follow RAFT's evaluate.py: Sintel is pooled over pixels without the max-flow test ('pixel'), KITTI is averaged
per image with Fl-all ('image'); chairs and things use the reference's Keras metric ('keras', max_flow 400).  Frames
are zero-padded to a multiple of 8 (the reference's CropOrPadder), not edge-replicated as in RAFT's InputPadder.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), '..')))

import tf_raft_b200 as T  # noqa: E402
from tf_raft_b200 import datasets as D  # noqa: E402

DEFAULTS = {'sintel': ('pixel', None), 'kitti': ('image', 400), 'chairs': ('keras', 400), 'things': ('keras', 400),
            'hd1k': ('image', 400)}


def dataset(name, args):
    if name == 'sintel':
        return D.MpiSintel(split='training', root=args.root, dstype=args.dstype)
    if name == 'kitti':
        return D.KITTI(split='training', root=args.root)
    if name == 'chairs':
        return D.FlyingChairs(split='validation', split_txt=args.split_txt, root=args.root)
    if name == 'things':
        return D.FlyingThings3D(root=args.root, dstype=args.dstype)
    return D.HD1K(root=args.root)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('dataset', choices=sorted(DEFAULTS))
    ap.add_argument('--root', required=True)
    ap.add_argument('--checkpoint', required=True, help='TF checkpoint prefix (the path before .index)')
    ap.add_argument('--small', action='store_true', help='SmallRAFT instead of RAFT')
    ap.add_argument('--dstype', default=None, help="Sintel 'clean' / 'final'; Things 'frames_cleanpass' / ...")
    ap.add_argument('--split-txt', default='FlyingChairs_train_val.txt')
    ap.add_argument('--iters', type=int, default=24)
    ap.add_argument('--batch-size', type=int, default=4)
    ap.add_argument('--workers', type=int, default=8)
    ap.add_argument('--protocol', choices=T.evaluation.PROTOCOLS, default=None)
    ap.add_argument('--max-flow', type=float, default=-1, help='ground-truth magnitude cut; 0 turns it off')
    args = ap.parse_args()
    if args.dstype is None:
        args.dstype = 'frames_cleanpass' if args.dataset == 'things' else 'clean'
    protocol, max_flow = DEFAULTS[args.dataset]
    protocol = args.protocol or protocol
    if args.max_flow >= 0:
        max_flow = args.max_flow or None
    model = (T.SmallRAFT if args.small else T.RAFT)(iters_pred=args.iters)
    model.load_params(T.load_tf_checkpoint(args.checkpoint, expect=model.state_dict()))
    ds = dataset(args.dataset, args)
    res = T.evaluate(model, ds, batch_size=args.batch_size, max_flow=max_flow, protocol=protocol, workers=args.workers)
    print(json.dumps({'dataset': args.dataset, 'pairs': len(ds), 'protocol': protocol, 'max_flow': max_flow,
                      'iters': args.iters, **res}))


if __name__ == '__main__':
    main()
