"""The RAFT forward entered from a warm start, coords1 = coords0 + flow_init (test infrastructure).

tf-raft has no warm start: its loop always starts from zero flow (model.py:89).  `forward` restates
oracle.raft_torch.forward for inference from raft_torch's own building blocks (encoders, CorrBlock, update blocks,
upsampling) with that one difference; flow_init=None gives raft_torch.forward's results exactly
(tests/test_video.py checks that).
"""
import torch
import torch.nn.functional as F

from . import raft_torch as rt


def forward(params, image1, image2, variant='raft', iters=12, dtype=torch.float32, flow_init=None,
            return_intermediates=False):
    """raft_torch.forward(..., training=False) with coords1 = coords0 + flow_init (B, H/8, W/8, 2) in `dtype`.
    Returns the `iters` NHWC predictions; with return_intermediates also the dict of per-iteration corr / coords and the
    corr_pyramid, as raft_torch.forward gives it."""
    cfg = rt.VARIANTS[variant]
    ops = rt.Ops(params, dtype)
    x1 = 2 * (rt._t(image1, dtype) / 255.0) - 1.0                          # model.py:70-71
    x2 = 2 * (rt._t(image2, dtype) / 255.0) - 1.0
    bs, H, W, _ = x1.shape
    fm = rt.encoder(ops, torch.cat([x1, x2], dim=0).permute(0, 3, 1, 2), 'fnet', cfg['fnorm'], False).permute(0, 2, 3, 1)
    fmap1, fmap2 = fm[:bs].contiguous(), fm[bs:].contiguous()             # :74
    corr_block = rt.CorrBlock(fmap1, fmap2, cfg['levels'], cfg['radius'])  # :77-79
    cnet = rt.encoder(ops, x1.permute(0, 3, 1, 2), 'cnet', cfg['cnorm'], False)   # :82
    net = torch.tanh(cnet[:, :cfg['hidden']])                              # :84-86
    inp = F.relu(cnet[:, cfg['hidden']:])
    coords0 = rt.coords_grid(bs, H // 8, W // 8, dtype)                    # :89
    coords1 = coords0.clone() if flow_init is None else coords0 + rt._t(flow_init, dtype)
    block = rt.basic_update_block if variant == 'raft' else rt.small_update_block
    inter = dict(corr=[], coords=[], corr_pyramid=corr_block.corr_pyramid)
    preds = []
    for _ in range(iters):                                                 # :93
        corr = corr_block.retrieve(coords1)                                # :95
        flow = coords1 - coords0                                           # :97
        net, mask, delta = block(ops, net, inp, corr.permute(0, 3, 1, 2), flow.permute(0, 3, 1, 2))
        coords1 = coords1 + delta.permute(0, 2, 3, 1)                      # :102
        if variant == 'raft':
            preds.append(rt.upsample_flow(coords1 - coords0, mask.permute(0, 2, 3, 1)))   # :105
        else:
            preds.append(rt.upflow8(coords1 - coords0))                   # :223
        inter['corr'].append(corr)
        inter['coords'].append(coords1)
    return (preds, inter) if return_intermediates else preds
