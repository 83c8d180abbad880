"""Losses / metrics -- host-side mirror of tf_raft/losses/losses.py (torch elementwise ops; not on
the hot path).  `y_true = (flow_gt, valid)`, predictions NHWC.  UnsupervisedLoss, an addition, runs in CUDA."""
import torch
import torch.distributed as dist

from . import _lib
from .layers.corr import fb_occlusion


def _valid_mask(flow_gt, valid, max_flow):
    mag = torch.sqrt(torch.sum(flow_gt ** 2, dim=-1))
    return valid.to(torch.bool) & (mag < max_flow)


def sequence_loss(y_true, y_pred, gamma=0.8, max_flow=400):
    """Reference losses.py:4-21: gamma-weighted L1 over the prediction sequence."""
    flow_gt, valid = y_true
    flow_gt = torch.as_tensor(flow_gt, dtype=torch.float32)
    valid = _valid_mask(flow_gt, torch.as_tensor(valid, device=flow_gt.device), max_flow)
    valid = valid.to(torch.float32).unsqueeze(-1)
    n = len(y_pred)
    loss = 0.0
    for i in range(n):
        w = gamma ** (n - i - 1)
        pred = torch.as_tensor(y_pred[i], dtype=torch.float32, device=flow_gt.device)
        loss = loss + w * torch.mean(valid * torch.abs(pred - flow_gt))
    return loss


def end_point_error(y_true, y_pred, max_flow=400):
    """Reference losses.py:24-43: epe and the <1 / <3 / <5 px rates over valid pixels."""
    flow_gt, valid = y_true
    flow_gt = torch.as_tensor(flow_gt, dtype=torch.float32)
    valid = _valid_mask(flow_gt, torch.as_tensor(valid, device=flow_gt.device), max_flow)
    pred = torch.as_tensor(y_pred, dtype=torch.float32, device=flow_gt.device)
    epe = torch.sqrt(torch.sum((pred - flow_gt) ** 2, dim=-1))[valid]
    return {'epe': epe.mean(), 'u1': (epe < 1).float().mean(), 'u3': (epe < 3).float().mean(),
            'u5': (epe < 5).float().mean()}


class EndPointError:
    """Reference losses.py:46-85: the streaming metric -- per update the means of epe / <1 / <3 / <5 px over the valid
    pixels of the LAST prediction are accumulated; result() is their average over the updates."""

    def __init__(self, max_flow=400, **kwargs):
        self.max_flow = max_flow
        self.reset_states()

    def reset_states(self):
        self.epe = self.u1 = self.u3 = self.u5 = 0.0
        self.count = 0

    def update_state(self, y_true, y_pred):
        info = end_point_error(y_true, y_pred[-1], self.max_flow)
        self.epe += float(info['epe'])
        self.u1 += float(info['u1'])
        self.u3 += float(info['u3'])
        self.u5 += float(info['u5'])
        self.count += 1

    def result(self):
        n = max(self.count, 1)
        return {'epe': self.epe / n, 'u1': self.u1 / n, 'u3': self.u3 / n, 'u5': self.u5 / n}


# ------------------------------------------------------------------------------------------------ self-supervised
def census_transform(images):
    """Census features of (B, H, W, 3) float images in 0..255 on the GPU -> (B, H, W, 48) float32 (raft_b200_census):
    channel k of pixel (x, y) is t / sqrt(0.81 + t^2), t the grey-value difference to the k-th neighbour of the 7 x 7
    window in row-major order, grey = (0.2989 R + 0.5870 G + 0.1140 B) / 255 and 0 outside the frame."""
    images = _lib.f32c(images)
    if images.dim() != 4 or images.shape[-1] != 3:
        raise ValueError(f'census_transform: expected (B, H, W, 3) images, got {tuple(images.shape)}')
    b, h, w, _ = images.shape
    out = torch.empty((b, h, w, 48), dtype=torch.float32, device=images.device)
    _lib.call('census', images.device, _lib.ptr(images), b, h, w, _lib.ptr(out))
    return out


class UnsupervisedLoss:
    """Self-supervised loss of bidirectional predictions, for training without ground truth (an addition: tf-raft
    trains on labelled flow only).  Given images I1, I2 (B, H, W, 3) in 0..255 and the n predictions of each direction,
    fw (I1 -> I2) and bw (I2 -> I1):

      L = census_weight * (L_c,fw + L_c,bw) / 2 + smoothness_weight * (L_s,fw + L_s,bw) / 2

    * L_c,d = sum_i gamma^(n-1-i) sum_x m(x) (D_i(x) + 0.01)^0.4 / max(sum_x m, 1): D_i(x) = sum_c d^2 / (0.1 + d^2),
      d the difference between the census of the target image at x and the bilinear sample of the source image's census
      at x + F_i(x); a landing outside the frame contributes 0.  m(x) is 1 where the pixel is at least 3 px from every
      border and not occluded by `fb_occlusion(F_fw[-1], F_bw[-1], alpha1, alpha2)` on the detached final predictions.
    * L_s,d = sum_i gamma^(n-1-i) (S_h + S_v) / 2, S_h (S_v) the mean over horizontal (vertical) neighbour pairs of
      exp(-edge_weight * mean_c |I_c(x') - I_c(x)| / 255) (|dFx| + |dFy|) / 2, edge-aware first-order smoothness.

    The census is computed once per image per call and carries no gradient; gradients reach the predictions only.  The
    loss and its gradient with respect to every prediction come from one CUDA pass per direction
    (raft_b200_unsup_loss, DESIGN.md section 9.1), deterministic: two calls on the same inputs give the same bits.

    Under torch.distributed with R ranks, each holding an equal shard of the batch, the census sums of every rank are
    normalised by the mask count C of the whole batch (one all-reduce of the two directions' counts): rank r's loss is
    census_weight (sum_{x in r} m rho) R / max(C, 1) / 2 per direction plus its smoothness share, so the mean of the
    ranks' losses is the whole batch's loss and the gradients summed over the ranks and divided by R are the whole
    batch's gradient.

    The defaults are untuned starting values, not settings validated on any dataset.  `compile(loss=UnsupervisedLoss())`
    makes `train_step` run the bidirectional training graph on (image1, image2[, flow, valid]) batches."""

    def __init__(self, census_weight=1.0, smoothness_weight=0.5, edge_weight=150.0, gamma=0.8, alpha1=0.01, alpha2=0.5):
        for name, v in (('census_weight', census_weight), ('smoothness_weight', smoothness_weight),
                        ('edge_weight', edge_weight), ('gamma', gamma), ('alpha1', alpha1), ('alpha2', alpha2)):
            if not (0.0 <= float(v) < float('inf')):
                raise ValueError(f'UnsupervisedLoss: {name} must be finite and >= 0, got {v}')
        self.census_weight, self.smoothness_weight = float(census_weight), float(smoothness_weight)
        self.edge_weight, self.gamma = float(edge_weight), float(gamma)
        self.alpha1, self.alpha2 = float(alpha1), float(alpha2)

    def __call__(self, images, preds):
        """images = (image1, image2), each (B, H, W, 3); preds = (preds_fw, preds_bw), each a list of n (B, H, W, 2)
        predictions (what `TrainGraph.forward_bidirectional` returns).  Returns the scalar loss (float32 tensor)."""
        from . import train
        image1, image2 = images
        preds_fw, preds_bw = list(preds[0]), list(preds[1])
        if not preds_fw or len(preds_fw) != len(preds_bw):
            raise ValueError(f'UnsupervisedLoss: {len(preds_fw)} forward and {len(preds_bw)} backward predictions')
        with torch.no_grad():
            occ = torch.cat(fb_occlusion(preds_fw[-1].detach(), preds_bw[-1].detach(), self.alpha1, self.alpha2))
            images = torch.cat([image1, image2]).to(torch.float32).contiguous()
            census = census_transform(images)
            census_norm = None
            if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
                h, w = occ.shape[1:]                                           # m: not occluded, 3 px inside the frame
                counts = (~occ[:, 3:h - 3, 3:w - 3]).reshape(2, -1).sum(1).to(torch.float64)
                dist.all_reduce(counts)                                          # the whole batch's (fw, bw) counts
                census_norm = counts.clamp(min=1.0) / dist.get_world_size()
        flows = torch.stack(preds_fw + preds_bw)                                 # (2n, B, H, W, 2)
        args = (flows, census, images, occ, self.census_weight, self.smoothness_weight, self.edge_weight, self.gamma)
        return train._UnsupLoss.apply(*args, *(() if census_norm is None else (census_norm,)))
