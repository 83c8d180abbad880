"""The original RAFT's training augmentors (core/utils/augmentor.py) restated on the real torchvision ColorJitter, PIL
and cv2 (test infrastructure; needs torchvision, Pillow and OpenCV).

FlowAugmentor / SparseFlowAugmentor draw from the same generators in the same order as RAFT's classes: np.random for the
asymmetric gate, the eraser and the spatial steps, torch's default CPU generator inside ColorJitter.  Seeding both and
calling either these or tf_raft_b200's augmentors with colour='torchvision' gives the same parameters, so the GPU
output can be compared with these byte for byte.

`__call__` returns RAFT's own results: uint8 images and the dense flow in float64 (the product of `flow * [sx, sy]`),
or for the sparse augmentor a float32 flow and an int32 valid.  `ReplayJitter` is a ColorJitter whose get_params
returns given draws, for tests that pin the op order.
"""
import cv2
import numpy as np
import torch
from PIL import Image
from torchvision.transforms import ColorJitter

cv2.setNumThreads(0)


class ReplayJitter(ColorJitter):
    """ColorJitter whose forward applies `draws` = [(order, b, c, s, h), ...] in turn instead of drawing."""

    def __init__(self, draws):
        super().__init__()
        self.draws = list(draws)

    def get_params(self, *_):
        order, b, c, s, h = self.draws.pop(0)
        return torch.tensor(order), b, c, s, h


def _jitter(photo_aug, img):
    return np.array(photo_aug(Image.fromarray(img)), dtype=np.uint8)


def _eraser(aug, img1, img2, bounds=(50, 100)):
    ht, wd = img1.shape[:2]
    if np.random.rand() < aug.eraser_aug_prob:
        mean_color = np.mean(img2.reshape(-1, 3), axis=0)
        for _ in range(np.random.randint(1, 3)):
            x0 = np.random.randint(0, wd)
            y0 = np.random.randint(0, ht)
            dx = np.random.randint(bounds[0], bounds[1])
            dy = np.random.randint(bounds[0], bounds[1])
            img2[y0:y0 + dy, x0:x0 + dx, :] = mean_color
    return img1, img2


def _resize(img, sx, sy):
    return cv2.resize(img, None, fx=sx, fy=sy, interpolation=cv2.INTER_LINEAR)


class FlowAugmentor:
    def __init__(self, crop_size, min_scale=-0.2, max_scale=0.5, do_flip=True):
        self.crop_size = crop_size
        self.min_scale, self.max_scale = min_scale, max_scale
        self.spatial_aug_prob, self.stretch_prob, self.max_stretch = 0.8, 0.8, 0.2
        self.do_flip, self.h_flip_prob, self.v_flip_prob = do_flip, 0.5, 0.1
        self.photo_aug = ColorJitter(brightness=0.4, contrast=0.4, saturation=0.4, hue=0.5 / 3.14)
        self.asymmetric_color_aug_prob = 0.2
        self.eraser_aug_prob = 0.5

    def color_transform(self, img1, img2):
        if np.random.rand() < self.asymmetric_color_aug_prob:
            return _jitter(self.photo_aug, img1), _jitter(self.photo_aug, img2)
        stack = _jitter(self.photo_aug, np.concatenate([img1, img2], axis=0))
        return tuple(np.split(stack, 2, axis=0))

    def spatial_transform(self, img1, img2, flow):
        ht, wd = img1.shape[:2]
        min_scale = np.maximum((self.crop_size[0] + 8) / float(ht), (self.crop_size[1] + 8) / float(wd))
        scale = 2 ** np.random.uniform(self.min_scale, self.max_scale)
        scale_x = scale_y = scale
        if np.random.rand() < self.stretch_prob:
            scale_x *= 2 ** np.random.uniform(-self.max_stretch, self.max_stretch)
            scale_y *= 2 ** np.random.uniform(-self.max_stretch, self.max_stretch)
        scale_x = np.clip(scale_x, min_scale, None)
        scale_y = np.clip(scale_y, min_scale, None)
        if np.random.rand() < self.spatial_aug_prob:
            img1, img2 = _resize(img1, scale_x, scale_y), _resize(img2, scale_x, scale_y)
            flow = _resize(flow, scale_x, scale_y) * [scale_x, scale_y]
        if self.do_flip:
            if np.random.rand() < self.h_flip_prob:
                img1, img2, flow = img1[:, ::-1], img2[:, ::-1], flow[:, ::-1] * [-1.0, 1.0]
            if np.random.rand() < self.v_flip_prob:
                img1, img2, flow = img1[::-1, :], img2[::-1, :], flow[::-1, :] * [1.0, -1.0]
        y0 = np.random.randint(0, img1.shape[0] - self.crop_size[0])
        x0 = np.random.randint(0, img1.shape[1] - self.crop_size[1])
        sl = np.s_[y0:y0 + self.crop_size[0], x0:x0 + self.crop_size[1]]
        return img1[sl], img2[sl], flow[sl]

    def __call__(self, img1, img2, flow):
        img1, img2 = self.color_transform(img1, img2)
        img1, img2 = _eraser(self, img1, img2)
        img1, img2, flow = self.spatial_transform(img1, img2, flow)
        return np.ascontiguousarray(img1), np.ascontiguousarray(img2), np.ascontiguousarray(flow)


class SparseFlowAugmentor:
    def __init__(self, crop_size, min_scale=-0.2, max_scale=0.5, do_flip=False):
        self.crop_size = crop_size
        self.min_scale, self.max_scale = min_scale, max_scale
        self.spatial_aug_prob = 0.8
        self.do_flip = do_flip
        self.photo_aug = ColorJitter(brightness=0.3, contrast=0.3, saturation=0.3, hue=0.3 / 3.14)
        self.eraser_aug_prob = 0.5

    def color_transform(self, img1, img2):
        stack = _jitter(self.photo_aug, np.concatenate([img1, img2], axis=0))
        return tuple(np.split(stack, 2, axis=0))

    @staticmethod
    def resize_sparse_flow_map(flow, valid, fx=1.0, fy=1.0):
        ht, wd = flow.shape[:2]
        coords = np.stack(np.meshgrid(np.arange(wd), np.arange(ht)), axis=-1).reshape(-1, 2).astype(np.float32)
        flow = flow.reshape(-1, 2).astype(np.float32)
        valid = valid.reshape(-1).astype(np.float32)
        coords0, flow0 = coords[valid >= 1], flow[valid >= 1]
        ht1, wd1 = int(round(ht * fy)), int(round(wd * fx))
        coords1 = coords0 * [fx, fy]
        flow1 = flow0 * [fx, fy]
        xx = np.round(coords1[:, 0]).astype(np.int32)
        yy = np.round(coords1[:, 1]).astype(np.int32)
        v = (xx > 0) & (xx < wd1) & (yy > 0) & (yy < ht1)
        flow_img = np.zeros([ht1, wd1, 2], dtype=np.float32)
        valid_img = np.zeros([ht1, wd1], dtype=np.int32)
        flow_img[yy[v], xx[v]] = flow1[v]
        valid_img[yy[v], xx[v]] = 1
        return flow_img, valid_img

    def spatial_transform(self, img1, img2, flow, valid):
        ht, wd = img1.shape[:2]
        min_scale = np.maximum((self.crop_size[0] + 1) / float(ht), (self.crop_size[1] + 1) / float(wd))
        scale = 2 ** np.random.uniform(self.min_scale, self.max_scale)
        scale_x = np.clip(scale, min_scale, None)
        scale_y = np.clip(scale, min_scale, None)
        if np.random.rand() < self.spatial_aug_prob:
            img1, img2 = _resize(img1, scale_x, scale_y), _resize(img2, scale_x, scale_y)
            flow, valid = self.resize_sparse_flow_map(flow, valid, fx=scale_x, fy=scale_y)
        if self.do_flip and np.random.rand() < 0.5:
            img1, img2, flow, valid = img1[:, ::-1], img2[:, ::-1], flow[:, ::-1] * [-1.0, 1.0], valid[:, ::-1]
        margin_y, margin_x = 20, 50
        y0 = np.random.randint(0, img1.shape[0] - self.crop_size[0] + margin_y)
        x0 = np.random.randint(-margin_x, img1.shape[1] - self.crop_size[1] + margin_x)
        y0 = np.clip(y0, 0, img1.shape[0] - self.crop_size[0])
        x0 = np.clip(x0, 0, img1.shape[1] - self.crop_size[1])
        sl = np.s_[y0:y0 + self.crop_size[0], x0:x0 + self.crop_size[1]]
        return img1[sl], img2[sl], flow[sl], valid[sl]

    def __call__(self, img1, img2, flow, valid):
        img1, img2 = self.color_transform(img1, img2)
        img1, img2 = _eraser(self, img1, img2)
        img1, img2, flow, valid = self.spatial_transform(img1, img2, flow, valid)
        return (np.ascontiguousarray(img1), np.ascontiguousarray(img2), np.ascontiguousarray(flow),
                np.ascontiguousarray(valid))
