"""Write a Sintel or KITTI benchmark submission from a TF checkpoint of tf-raft, in RAFT's file layout.

    python scripts/submit.py sintel --root datasets/MPI-Sintel-complete --checkpoint checkpoints/model --out submission
    python scripts/submit.py kitti --root datasets/KITTI --checkpoint checkpoints/model --out submission/flow

Sintel: `<out>/<clean|final>/<scene>/frame%04d.flo` for the test split, warm-started scene by scene unless
`--no-warm-start`.  KITTI: `<out>/<frame_id>` 16-bit flow PNGs for the testing split.  Frames are edge-replicated to a
multiple of 8 (RAFT's InputPadder).  The iteration counts default to RAFT's: 32 for Sintel, 24 for KITTI.  Prints one
JSON line.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), '..')))

import tf_raft_b200 as T  # noqa: E402

ITERS = {'sintel': 32, 'kitti': 24}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('dataset', choices=sorted(ITERS))
    ap.add_argument('--root', required=True)
    ap.add_argument('--checkpoint', required=True, help='TF checkpoint prefix (the path before .index)')
    ap.add_argument('--out', required=True)
    ap.add_argument('--iters', type=int, default=None, help='update iterations (default: 32 Sintel, 24 KITTI)')
    ap.add_argument('--no-warm-start', action='store_true', help='Sintel: predict every pair from zero flow')
    ap.add_argument('--small', action='store_true', help='SmallRAFT instead of RAFT')
    ap.add_argument('--workers', type=int, default=4)
    args = ap.parse_args()
    iters = args.iters or ITERS[args.dataset]
    model = (T.SmallRAFT if args.small else T.RAFT)(iters_pred=iters)
    model.load_params(T.load_tf_checkpoint(args.checkpoint, expect=model.state_dict()))
    if args.dataset == 'sintel':
        n = T.create_sintel_submission(model, args.root, args.out, warm_start=not args.no_warm_start,
                                       workers=args.workers)
    else:
        n = T.create_kitti_submission(model, args.root, args.out, workers=args.workers)
    print(json.dumps({'dataset': args.dataset, 'files': n, 'iters': iters, 'out': args.out,
                      'warm_start': args.dataset == 'sintel' and not args.no_warm_start}))


if __name__ == '__main__':
    main()
