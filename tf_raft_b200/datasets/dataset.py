"""The reference's datasets (tf_raft/datasets/dataset.py:20-268): FlowDataset and MpiSintel, FlyingChairs,
FlyingThings3D, KITTI and HD1K, with the reference's names, arguments, defaults and file lists.

`__getitem__` is the reference's per-item contract on the host, returning NumPy arrays.  The one difference: with
`aug_params` the item goes through this package's GPU FlowAugmentor / SparseFlowAugmentor and comes back as CUDA
tensors.  It serves VisFlowCallback and single items; `FlowDataset.batches` is the fast path, a thread-pool loader that
hands batches to the GPU (KITTI / HD1K flow PNGs are decoded there, csrc/dataset.cuh).

Not ported: `fetch_dataloader` (:271-306; it calls an undefined `data.DataLoader`) and `ShapeSetter` (:309-316), which
only sets static shapes on TensorFlow tensors.  `CropOrPadder` is `tf_raft_b200.preprocess.CropOrPadder`.
"""
import collections
import concurrent.futures
import copy
import os
import os.path as osp
from glob import glob

import numpy as np
import torch

from ..preprocess import resize_with_crop_or_pad
from . import frame_utils
from .augmentor import FlowAugmentor, SparseFlowAugmentor
from .png16 import check_png16_status, decode_png16


def _frame(path):
    """dataset.py:72-85 for one frame: uint8, grayscale tiled to 3 channels, RGBA cut to RGB."""
    img = np.array(frame_utils.read_gen(path)).astype(np.uint8)
    return np.tile(img[..., None], (1, 1, 3)) if img.ndim == 2 else img[..., :3]


def _dense_valid(flow):
    """dataset.py:102: |u| < 1000 and |v| < 1000 (bool)."""
    return (np.abs(flow[:, :, 0]) < 1000) * (np.abs(flow[:, :, 1]) < 1000)


class FlowDataset:
    """dataset.py:20-129.  Container quirks kept from the reference:

    - `2 * ds` and `a + b` (`__rmul__`, `__add__`) repeat or extend `flow_list` and `image_list` only; `extra_info`
      is left as it was.
    - `a + b` keeps the LEFT operand's augmentor and `sparse` flag: `sintel + kitti` reads KITTI's flows as dense.
    - `shuffle()` draws `np.random.permutation(len(self))`, so a seeded run shuffles as the reference does (and it
      leaves `extra_info` in place too).
    - `__call__` yields `self[0], self[1], ...`.  For a training dataset this never ends, because `__getitem__` takes
      `index % len` (:65); the reference bounds it with `steps_per_epoch` / `validation_steps`.  A test dataset stops at
      its end.
    """

    def __init__(self, aug_params=None, sparse=False):
        self.augmentor = None
        self.sparse = sparse
        if aug_params is not None:
            self.augmentor = (SparseFlowAugmentor if sparse else FlowAugmentor)(**aug_params)
        self.is_test = False
        self.init_seed = False
        self.flow_list = []
        self.image_list = []
        self.extra_info = []

    def __getitem__(self, index):
        """Test datasets: (img1, img2, extra_info).  Otherwise (img1 uint8 (H, W, 3), img2, flow float32 (H, W, 2),
        valid): a bool dense valid (:102) or KITTI's float32 B channel (sparse).  With an augmentor: the augmentor's
        CUDA tensors (img1, img2, flow, valid float32), valid taken on the fp64 flow as in `FlowAugmentor.batch`."""
        if self.is_test:
            return _frame(self.image_list[index][0]), _frame(self.image_list[index][1]), self.extra_info[index]
        index = index % len(self.image_list)
        valid = None
        if self.sparse:
            flow, valid = frame_utils.read_flow_kitti(self.flow_list[index])
        else:
            flow = frame_utils.read_gen(self.flow_list[index])
        img1, img2 = _frame(self.image_list[index][0]), _frame(self.image_list[index][1])
        flow = np.array(flow).astype(np.float32)
        if self.augmentor is not None:
            sample = (img1, img2, flow, valid) if self.sparse else (img1, img2, flow)
            return tuple(t[0] for t in self.augmentor.batch([sample]))
        return img1, img2, flow, (valid if valid is not None else _dense_valid(flow))

    def __rmul__(self, v):
        self_copy = copy.deepcopy(self)
        self_copy.flow_list *= v
        self_copy.image_list *= v
        return self_copy

    def __add__(self, other):
        copied = copy.deepcopy(self)
        copied.flow_list += other.flow_list
        copied.image_list += other.image_list
        return copied

    def __len__(self):
        return len(self.image_list)

    def __call__(self):
        for sample in self:
            yield sample

    def shuffle(self):
        perm = np.random.permutation(len(self))
        self.flow_list = [self.flow_list[i] for i in perm]
        self.image_list = [self.image_list[i] for i in perm]

    # ------------------------------------------------------------------ the batch loader
    def _load(self, index):
        """Worker side of `batches`: the host reads of one item.  No random draws happen here."""
        img1, img2 = _frame(self.image_list[index][0]), _frame(self.image_list[index][1])
        if self.is_test:
            return img1, img2, None, None
        path = self.flow_list[index]
        if self.sparse:
            return img1, img2, ('png16', path, frame_utils.inflate_png16(path)), None
        flow = np.array(frame_utils.read_gen(path)).astype(np.float32)
        valid = None if self.augmentor is not None else _dense_valid(flow).astype(np.float32)
        return img1, img2, flow, valid

    def batches(self, batch_size, *, target_size=None, workers=4, device=None, drop_last=False):
        """Batches of the items in index order, read by `workers` threads ahead of the consumer.

        Training mode (the dataset has an augmentor): yields `(image1, image2, flow, valid)` CUDA batches from
        `augmentor.batch`, ready for `RAFT.train_step`.  The augmentation parameters are drawn on the consuming thread
        in item order, so seeding `np.random` and `random` as the reference does gives the reference's parameter stream.

        Evaluation mode (no augmentor): yields `(image1, image2, flow, valid, sizes)`: uint8 frames and float32 flow /
        valid crop-or-padded to `target_size` as `CropOrPadder` does (zero padding; padded pixels invalid), and each
        item's original (H, W).  With `target_size=None` each item gets the smallest centred padding to a multiple of 8,
        and a batch closes early when the padded shape changes.  Test datasets yield flow = valid = None.

        Host buffers are pinned; the upload of a batch runs on a copy stream and overlaps the consumer's GPU work."""
        if batch_size < 1:
            raise ValueError('batch_size must be >= 1')
        if self.is_test and self.augmentor is not None:
            raise ValueError('a test dataset has no flows to augment')
        device = torch.device(device if device is not None else
                              (self.augmentor.device if self.augmentor is not None else 'cuda'))
        if device.type != 'cuda':
            raise RuntimeError('FlowDataset.batches feeds CUDA tensors only (sm_90a); there is no CPU fallback')
        up = _Uploader(device)
        with concurrent.futures.ThreadPoolExecutor(max(1, int(workers))) as pool:
            ahead = collections.deque()
            nxt, n = 0, len(self)
            depth = max(2 * batch_size, 2 * max(1, int(workers)))

            def take():
                nonlocal nxt
                while nxt < n and len(ahead) < depth:
                    ahead.append(pool.submit(self._load, nxt))
                    nxt += 1
                return ahead.popleft().result() if ahead else None

            if self.augmentor is not None:
                while True:
                    items = []
                    while len(items) < batch_size:
                        item = take()
                        if item is None:
                            break
                        items.append(item)
                    if not items or (drop_last and len(items) < batch_size):
                        break
                    samples = up.stage(items)
                    out = self.augmentor.batch([s[:4] if self.sparse else s[:3] for s in samples])
                    up.release()
                    yield out
                    if len(items) < batch_size:
                        break
            else:
                pending = take()
                while pending is not None:
                    shape = self._padded(pending[0].shape[:2], target_size)
                    items = [pending]
                    pending = take()
                    while pending is not None and len(items) < batch_size and \
                            self._padded(pending[0].shape[:2], target_size) == shape:
                        items.append(pending)
                        pending = take()
                    if drop_last and len(items) < batch_size:
                        continue
                    yield self._eval_batch(up, items, shape)
        up.finish()

    @staticmethod
    def _padded(hw, target_size):
        if target_size is not None:
            return tuple(int(s) for s in target_size)
        return tuple(-(-int(s) // 8) * 8 for s in hw)

    def _eval_batch(self, up, items, shape):
        th, tw = shape
        samples = up.stage(items)
        img1 = torch.stack([resize_with_crop_or_pad(s[0], th, tw) for s in samples])
        img2 = torch.stack([resize_with_crop_or_pad(s[1], th, tw) for s in samples])
        flow = valid = None
        if not self.is_test:
            flow = torch.stack([resize_with_crop_or_pad(s[2], th, tw) for s in samples])
            valid = torch.stack([resize_with_crop_or_pad(s[3].unsqueeze(-1), th, tw).squeeze(-1) for s in samples])
        up.release()
        return img1, img2, flow, valid, [tuple(it[0].shape[:2]) for it in items]


class _Uploader:
    """One pinned host buffer -> one device buffer per batch, two of each in turn.  A host buffer is refilled only after
    its copy has finished, a device buffer only after the work that read it (enqueued before `release`) has run."""

    def __init__(self, device):
        self.device = device
        self.copy = torch.cuda.Stream(device=device)
        self.host = [None, None]
        self.dev = [None, None]
        self.copied = [None, None]
        self.freed = [None, None]
        self.status = []                    # (pinned status, names, copy event) of PNG decodes not yet checked
        self.k = 1

    def stage(self, items):
        """items: worker outputs -> per item (img1, img2, flow, valid) device tensors (None stays None); 16-bit PNG
        flows are decoded on the device."""
        self.k ^= 1
        k, arrays, layout, off = self.k, [], [], 0
        for it in items:
            for a in it:
                if a is None:
                    continue
                if isinstance(a, tuple):                          # ('png16', path, (rows, h, w))
                    buf = np.frombuffer(a[2][0], dtype=np.uint8)
                else:
                    buf = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
                arrays.append((off, buf))
                layout.append(off)
                off += -(-buf.size // 16) * 16
        if self.copied[k] is not None:
            self.copied[k].synchronize()
        if self.host[k] is None or self.host[k].numel() < off:
            self.host[k] = torch.empty(max(off, 16), dtype=torch.uint8, pin_memory=True)
        hv = self.host[k].numpy()
        for o, buf in arrays:
            hv[o:o + buf.size] = buf
        main = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.copy):
            if self.freed[k] is not None:
                self.copy.wait_event(self.freed[k])
            if self.dev[k] is None or self.dev[k].numel() < off:
                self.dev[k] = torch.empty(max(off, 16), dtype=torch.uint8, device=self.device)
            self.dev[k][:off].copy_(self.host[k][:off], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.copy)
        self.copied[k] = ev
        main.wait_event(ev)
        dev = self.dev[k]
        out, pngs, j = [], [], 0
        for it in items:
            row = []
            for a in it:
                if a is None:
                    row.append(None)
                    continue
                o = layout[j]
                j += 1
                if isinstance(a, tuple):
                    _, path, (rows, h, w) = a
                    pngs.append((len(out), len(row), path, (o, h, w)))
                    row.extend([None, None])                      # flow and valid, filled below
                    continue
                t = dev[o:o + a.nbytes].view(torch.uint8 if a.dtype == np.uint8 else torch.float32)
                row.append(t.view(a.shape))
            out.append(row[:4])
        if pngs:
            status = torch.empty(len(pngs), dtype=torch.int32, pin_memory=True)
            decoded = decode_png16(dev, [p[3] for p in pngs], [p[2] for p in pngs], status_host=status)
            for (i, c, _, _), (flow, valid) in zip(pngs, decoded):
                out[i][c], out[i][c + 1] = flow, valid
            done = torch.cuda.Event()
            done.record(main)
            self.check()
            self.status.append((status, [p[2] for p in pngs], done))
        return out

    def release(self):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self.device))
        self.freed[self.k] = ev

    def check(self):
        """Raise for a PNG the kernel rejected, once its status has arrived (the host checks come first, so this
        only fires for a stream the host could not see into)."""
        keep = []
        for status, names, done in self.status:
            if done.query():
                check_png16_status(status, names)
            else:
                keep.append((status, names, done))
        self.status = keep

    def finish(self):
        for _, _, done in self.status:
            done.synchronize()
        self.check()


class MpiSintel(FlowDataset):
    """dataset.py:132-165, MPI Sintel.  Scenes come in `os.listdir` order (not sorted, as :158), frames sorted within
    a scene; extra_info = (scene, frame index); split='test' makes a test dataset."""

    def __init__(self, aug_params=None, split='training', root='datasets/MPI-Sintel-complete', dstype='clean'):
        super().__init__(aug_params)
        flow_root = osp.join(root, split, 'flow')
        image_root = osp.join(root, split, dstype)
        if split == 'test':
            self.is_test = True
        for scene in os.listdir(image_root):
            image_list = sorted(glob(osp.join(image_root, scene, '*.png')))
            for i in range(len(image_list) - 1):
                self.image_list += [[image_list[i], image_list[i + 1]]]
                self.extra_info += [(scene, i)]
            if split != 'test':
                self.flow_list += sorted(glob(osp.join(flow_root, scene, '*.flo')))


class FlyingChairs(FlowDataset):
    """dataset.py:168-200: sorted *.ppm / *.flo (asserting two frames per flow); `split_txt` read with np.loadtxt, code
    1 = training, 2 = validation."""

    def __init__(self, aug_params=None, split='training', split_txt='FlyingChairs_train_val.txt',
                 root='datasets/FlyingChairs_release/data'):
        super().__init__(aug_params)
        images = sorted(glob(osp.join(root, '*.ppm')))
        flows = sorted(glob(osp.join(root, '*.flo')))
        assert len(images) // 2 == len(flows)
        split_list = np.loadtxt(split_txt, dtype=np.int32)
        for i in range(len(flows)):
            xid = split_list[i]
            if (split == 'training' and xid == 1) or (split == 'validation' and xid == 2):
                self.flow_list += [flows[i]]
                self.image_list += [[images[2 * i], images[2 * i + 1]]]


class FlyingThings3D(FlowDataset):
    """dataset.py:203-227: the left camera; into_future pairs (i, i+1) with flow i, into_past (i+1, i) with flow i+1."""

    def __init__(self, aug_params=None, root='datasets/FlyingThings3D', dstype='frames_cleanpass'):
        super().__init__(aug_params)
        for cam in ['left']:
            for direction in ['into_future', 'into_past']:
                image_dirs = sorted(glob(osp.join(root, dstype, 'TRAIN/*/*')))
                image_dirs = sorted([osp.join(f, cam) for f in image_dirs])
                flow_dirs = sorted(glob(osp.join(root, 'optical_flow/TRAIN/*/*')))
                flow_dirs = sorted([osp.join(f, direction, cam) for f in flow_dirs])
                for idir, fdir in zip(image_dirs, flow_dirs):
                    images = sorted(glob(osp.join(idir, '*.png')))
                    flows = sorted(glob(osp.join(fdir, '*.pfm')))
                    for i in range(len(flows) - 1):
                        if direction == 'into_future':
                            self.image_list += [[images[i], images[i + 1]]]
                            self.flow_list += [flows[i]]
                        else:
                            self.image_list += [[images[i + 1], images[i]]]
                            self.flow_list += [flows[i + 1]]


class KITTI(FlowDataset):
    """dataset.py:230-249: image_2/*_10.png with *_11.png, flow_occ/*_10.png for training; extra_info = [frame file
    name]; split='testing' makes a test dataset.  Sparse: flows are 16-bit PNGs."""

    def __init__(self, aug_params=None, split='training', root='datasets/KITTI'):
        super().__init__(aug_params, sparse=True)
        if split == 'testing':
            self.is_test = True
        root = osp.join(root, split)
        images1 = sorted(glob(osp.join(root, 'image_2/*_10.png')))
        images2 = sorted(glob(osp.join(root, 'image_2/*_11.png')))
        for img1, img2 in zip(images1, images2):
            frame_id = img1.split('/')[-1]
            self.extra_info += [[frame_id]]
            self.image_list += [[img1, img2]]
        if split == 'training':
            self.flow_list = sorted(glob(osp.join(root, 'flow_occ/*_10.png')))


class HD1K(FlowDataset):
    """dataset.py:252-268: sequences %06d in turn until one has no flows; consecutive frames of a sequence."""

    def __init__(self, aug_params=None, root='datasets/HD1k'):
        super().__init__(aug_params, sparse=True)
        seq_ix = 0
        while 1:
            flows = sorted(glob(os.path.join(root, 'hd1k_flow_gt', 'flow_occ/%06d_*.png' % seq_ix)))
            images = sorted(glob(os.path.join(root, 'hd1k_input', 'image_2/%06d_*.png' % seq_ix)))
            if len(flows) == 0:
                break
            for i in range(len(flows) - 1):
                self.flow_list += [flows[i]]
                self.image_list += [[images[i], images[i + 1]]]
            seq_ix += 1


def as_supervised(image1, image2, flow, valid):
    """dataset.py:319-320."""
    return (image1, image2), (flow, valid)
