"""FlowAugmentor and SparseFlowAugmentor -- the reference's training augmentation (tf_raft/datasets/augmentor.py) on the
GPU, without OpenCV or albumentations.

Randomness lives on the host only: `sample_params` draws each sample's parameters from the reference's distributions
in the reference's call order, `np.random` for augmentor.py and Python's `random` for albumentations' gates and
get_params, so seeding both modules reproduces the reference's parameter stream.  The kernels
(raft_b200_augment_dense / _sparse, csrc/augment.cuh) take those parameters explicitly and reproduce cv2's uint8 and
float32 INTER_LINEAR resize and RGB<->HSV bit for bit (DESIGN.md section 3.5).
"""
import ctypes
import dataclasses
import random

import numpy as np
import torch

from .. import _lib


@dataclasses.dataclass
class AugmentParams:
    """One sample's random draws.  colourK = (bc, hsv) for image K: bc = (alpha, beta) of RandomBrightnessContrast or
    None when its gate is off, hsv = (hue, sat, val) shifts of HueSaturationValue or None.  rects: eraser rectangles
    (x0, y0, dx, dy) of img2 at source resolution.  spatial: resize by (scale_x, scale_y); then the flips and the crop
    window at (y0, x0) of the flipped, resized image."""
    colour1: tuple
    colour2: tuple
    rects: list
    scale_x: float
    scale_y: float
    spatial: bool
    hflip: bool
    vflip: bool
    y0: int
    x0: int
    crop: tuple


class _Sample(ctypes.Structure):
    """struct raft_augment_sample (include/raft_b200.h)."""
    _fields_ = [('img1', ctypes.c_void_p), ('img2', ctypes.c_void_p), ('flow', ctypes.c_void_p),
                ('valid', ctypes.c_void_p), ('out_img1', ctypes.c_void_p), ('out_img2', ctypes.c_void_p),
                ('out_flow', ctypes.c_void_p), ('out_valid', ctypes.c_void_p),
                ('scale_x', ctypes.c_double), ('scale_y', ctypes.c_double), ('ws_offset', ctypes.c_size_t),
                ('H', ctypes.c_int), ('W', ctypes.c_int), ('crop_h', ctypes.c_int), ('crop_w', ctypes.c_int),
                ('y0', ctypes.c_int), ('x0', ctypes.c_int), ('spatial', ctypes.c_int), ('hflip', ctypes.c_int),
                ('vflip', ctypes.c_int), ('hsv', ctypes.c_int * 2), ('n_rects', ctypes.c_int),
                ('rect', (ctypes.c_int * 4) * 2), ('lut', ((ctypes.c_uint8 * 256) * 4) * 2)]


# bc_lut and hsv_luts transcribe albumentations 0.4.6 (augmentations/functional.py, _brightness_contrast_adjust_uint and
# _shift_hsv_uint8), NumPy casting included; oracle/augment_np.py holds the tests' own transcription.
def bc_lut(alpha, beta):
    """albumentations 0.4.6 brightness_contrast_adjust on uint8 (brightness_by_max): float32 LUT, truncated."""
    lut = np.arange(0, 256).astype('float32')
    if alpha != 1:
        lut *= alpha
    if beta != 0:
        lut += beta * 255
    return np.clip(lut, 0, 255).astype(np.uint8)


def hsv_luts(hue_shift, sat_shift, val_shift):
    """albumentations 0.4.6 shift_hsv's LUTs on uint8: hue mod 180, sat and val clipped, truncated."""
    lut = np.arange(0, 256, dtype=np.int16)
    return (np.mod(lut + hue_shift, 180).astype(np.uint8), np.clip(lut + sat_shift, 0, 255).astype(np.uint8),
            np.clip(lut + val_shift, 0, 255).astype(np.uint8))


def resized_size(n, scale):
    """cv2.resize's output size for fx/fy = scale: round half to even."""
    return int(np.rint(np.float64(n) * np.float64(scale)))


class _Augmentor:
    _sparse = False

    def __init__(self, crop_size, min_scale, max_scale, do_flip, device):
        # spatial augmentation params
        self.crop_size = tuple(int(c) for c in crop_size)
        self.min_scale = min_scale
        self.max_scale = max_scale
        self.spatial_aug_prob = 0.8
        self.stretch_prob = 0.8
        self.max_stretch = 0.2
        # flip augmentation params
        self.do_flip = do_flip
        self.h_flip_prob = 0.5
        self.v_flip_prob = 0.1
        self.asymmetric_color_aug_prob = 0.2
        self.eraser_aug_prob = 0.5
        self.device = torch.device(device)

    # ---------------------------------------------------------------- the draws
    def _photo_params(self):
        """albumentations 0.4.6 Compose([RandomBrightnessContrast, HueSaturationValue]).__call__, every transform at its
        default p = 0.5 (read from 0.4.6's sources, core/composition.py and core/transforms_interface.py, not run):
        Compose draws random.random() < p (p = 1); each BasicTransform.__call__ draws random.random() < 0.5 and, if
        taken, its get_params: RandomBrightnessContrast alpha = 1 + uniform(contrast limits), beta = 0 +
        uniform(brightness limits); HueSaturationValue uniform hue, sat, val shifts (val's limit is 0, still drawn)."""
        bc_limit, (hue, sat, val) = self._photo_limits
        random.random()
        bc = hsv = None
        if random.random() < 0.5:
            alpha = 1.0 + random.uniform(-bc_limit, bc_limit)
            beta = 0.0 + random.uniform(-bc_limit, bc_limit)
            bc = (alpha, beta)
        if random.random() < 0.5:
            hsv = (random.uniform(-hue, hue), random.uniform(-sat, sat), random.uniform(-val, val))
        return bc, hsv

    def _eraser_params(self, ht, wd):
        """augmentor.py:61-74 (and :170-181)."""
        rects = []
        if np.random.rand() < self.eraser_aug_prob:
            for _ in range(np.random.randint(1, 3)):
                x0 = np.random.randint(0, wd)
                y0 = np.random.randint(0, ht)
                dx = np.random.randint(50, 100)
                dy = np.random.randint(50, 100)
                rects.append((int(x0), int(y0), int(dx), int(dy)))
        return rects

    def sample_params(self, ht, wd):
        """Draw one sample's AugmentParams for an (ht, wd) source, in the reference's call order.  Raises ValueError,
        as the reference's np.random.randint does, when the crop does not fit."""
        raise NotImplementedError

    # ---------------------------------------------------------------- the kernels
    def _prepare(self, sample):
        if len(sample) != (4 if self._sparse else 3):
            raise ValueError(f'{type(self).__name__}: expected {"(img1, img2, flow, valid)" if self._sparse else "(img1, img2, flow)"}')
        out = []
        for k, t in enumerate(sample):
            dtype = torch.uint8 if k < 2 else torch.float32
            if isinstance(t, np.ndarray):
                t = torch.from_numpy(np.ascontiguousarray(t, dtype=np.uint8 if k < 2 else np.float32)).to(self.device)
            if not isinstance(t, torch.Tensor) or not t.is_cuda:
                raise TypeError(f'{type(self).__name__}: inputs must be CUDA tensors or NumPy arrays')
            if t.device != self.device and self.device.index is not None:
                raise ValueError(f'{type(self).__name__}: input on {t.device}, augmentor on {self.device}')
            if k < 2 and t.dtype != torch.uint8:
                raise TypeError(f'{type(self).__name__}: images must be uint8')
            out.append(t.to(dtype).contiguous())
        img1, img2, flow = out[:3]
        h, w = img1.shape[:2]
        if img1.shape != (h, w, 3) or img2.shape != (h, w, 3) or flow.shape != (h, w, 2):
            raise ValueError(f'{type(self).__name__}: expected (H, W, 3) images and an (H, W, 2) flow, got '
                             f'{tuple(img1.shape)}, {tuple(img2.shape)}, {tuple(flow.shape)}')
        if self._sparse and out[3].shape != (h, w):
            raise ValueError(f'{type(self).__name__}: expected an (H, W) valid, got {tuple(out[3].shape)}')
        return out

    def _check(self, p, h, w):
        rh, rw = (resized_size(h, p.scale_y), resized_size(w, p.scale_x)) if p.spatial else (h, w)
        ch, cw = p.crop
        if not (0 <= p.y0 <= rh - ch and 0 <= p.x0 <= rw - cw):
            raise ValueError(f'{type(self).__name__}: crop {ch}x{cw} at ({p.y0}, {p.x0}) does not fit {rh}x{rw}')
        if (self._sparse and p.vflip) or len(p.rects) > 2:
            raise ValueError(f'{type(self).__name__}: unsupported parameters {p}')

    def batch(self, samples, params=None):
        """Augment a list of samples, of any source sizes, in one launch set.  samples: (img1, img2, flow) tuples
        (sparse: (img1, img2, flow, valid)), uint8 (H, W, 3) images and float32 (H, W, 2) flow as CUDA tensors (NumPy
        arrays are uploaded to `device`).  params: one AugmentParams per sample; drawn with sample_params by default.
        -> img1, img2 (B, ch, cw, 3) uint8, flow (B, ch, cw, 2) float32, valid (B, ch, cw) float32."""
        samples = [self._prepare(s) for s in samples]
        if not samples:
            raise ValueError(f'{type(self).__name__}.batch: no samples')
        if params is None:
            params = [self.sample_params(*s[0].shape[:2]) for s in samples]
        if len(params) != len(samples):
            raise ValueError(f'{type(self).__name__}.batch: {len(samples)} samples but {len(params)} parameter sets')
        crops = {tuple(p.crop) for p in params}
        if len(crops) != 1:
            raise ValueError(f'{type(self).__name__}.batch: one crop size per batch, got {sorted(crops)}')
        (ch, cw), b = crops.pop(), len(samples)
        dev = samples[0][0].device
        if any(t.device != dev for s in samples for t in s):
            raise ValueError(f'{type(self).__name__}.batch: every tensor of a batch must be on one device, '
                             f'got {sorted({str(t.device) for s in samples for t in s})}')
        img1 = torch.empty((b, ch, cw, 3), dtype=torch.uint8, device=dev)
        img2 = torch.empty_like(img1)
        flow = torch.empty((b, ch, cw, 2), dtype=torch.float32, device=dev)
        valid = torch.empty((b, ch, cw), dtype=torch.float32, device=dev)
        arr = (_Sample * b)()
        for i, (s, p) in enumerate(zip(samples, params)):
            h, w = s[0].shape[:2]
            self._check(p, h, w)
            a = arr[i]
            a.img1, a.img2, a.flow = s[0].data_ptr(), s[1].data_ptr(), s[2].data_ptr()
            a.valid = s[3].data_ptr() if self._sparse else None
            a.out_img1, a.out_img2 = img1[i].data_ptr(), img2[i].data_ptr()
            a.out_flow, a.out_valid = flow[i].data_ptr(), valid[i].data_ptr()
            a.scale_x, a.scale_y = float(p.scale_x), float(p.scale_y)
            a.H, a.W, a.crop_h, a.crop_w, a.y0, a.x0 = h, w, ch, cw, int(p.y0), int(p.x0)
            a.spatial, a.hflip, a.vflip = int(bool(p.spatial)), int(bool(p.hflip)), int(bool(p.vflip))
            for k, (bc, hsv) in enumerate((p.colour1, p.colour2)):
                luts = [bc_lut(*bc) if bc is not None else np.arange(256, dtype=np.uint8)]
                luts += list(hsv_luts(*hsv)) if hsv is not None else [np.arange(256, dtype=np.uint8)] * 3
                for j, lut in enumerate(luts):
                    ctypes.memmove(a.lut[k][j], lut.ctypes.data, 256)
                a.hsv[k] = int(hsv is not None)
            a.n_rects = len(p.rects)
            for r, rect in enumerate(p.rects):
                for j in range(4):
                    a.rect[r][j] = int(rect[j])
        nbytes = _lib.query_bytes('augment_workspace_bytes', arr, b, int(self._sparse))
        ws = _lib.workspace(nbytes, dev)
        arr_dev = torch.frombuffer(bytearray(arr), dtype=torch.uint8).to(dev)
        _lib.call('augment_sparse' if self._sparse else 'augment_dense', dev, arr, _lib.ptr(arr_dev), b, _lib.ptr(ws),
                  nbytes)
        return img1, img2, flow, valid


class FlowAugmentor(_Augmentor):
    """Reference augmentor.py:9-129 on the GPU.  Colour: albumentations 0.4.6 RandomBrightnessContrast(0.4, 0.4) then
    HueSaturationValue(28, 102, 0), one parameter set for both images, or (p = 0.2) one each.  Eraser (p = 0.5): one
    or two rectangles of img2 set to its mean colour.  Spatial: 2**uniform(min_scale, max_scale), stretched (p = 0.8)
    by 2**uniform(+-0.2) per axis, clipped to (crop + 8) / size, applied (p = 0.8) with cv2.resize INTER_LINEAR to
    both images and the flow, the flow then times (scale_x, scale_y) in fp64.  Flips (p = 0.5 h, 0.1 v) and a random
    crop.  The dense valid of dataset.py:102, |f| < 1000 per component, is taken on the fp64 flow."""
    _photo_limits = (0.4, (int(0.5 / 3.14 * 180), int(0.4 * 255), int(0.)))

    def __init__(self, crop_size, min_scale=-0.2, max_scale=0.5, do_flip=True, device='cuda'):
        super().__init__(crop_size, min_scale, max_scale, do_flip, device)

    def sample_params(self, ht, wd):
        if np.random.rand() < self.asymmetric_color_aug_prob:           # :46
            colour1 = self._photo_params()
            colour2 = self._photo_params()
        else:
            colour1 = colour2 = self._photo_params()
        rects = self._eraser_params(ht, wd)
        min_scale = np.maximum((self.crop_size[0] + 8) / float(ht), (self.crop_size[1] + 8) / float(wd))    # :79
        scale = 2 ** np.random.uniform(self.min_scale, self.max_scale)
        scale_x = scale
        scale_y = scale
        if np.random.rand() < self.stretch_prob:
            scale_x *= 2 ** np.random.uniform(-self.max_stretch, self.max_stretch)
            scale_y *= 2 ** np.random.uniform(-self.max_stretch, self.max_stretch)
        scale_x = np.clip(scale_x, min_scale, None)
        scale_y = np.clip(scale_y, min_scale, None)
        spatial = np.random.rand() < self.spatial_aug_prob
        hflip = vflip = False
        if self.do_flip:
            hflip = np.random.rand() < self.h_flip_prob
            vflip = np.random.rand() < self.v_flip_prob
        h1, w1 = (resized_size(ht, scale_y), resized_size(wd, scale_x)) if spatial else (ht, wd)
        y0 = np.random.randint(0, h1 - self.crop_size[0])                # :111
        x0 = np.random.randint(0, w1 - self.crop_size[1])
        return AugmentParams(colour1, colour2, rects, float(scale_x), float(scale_y), bool(spatial), bool(hflip),
                             bool(vflip), int(y0), int(x0), self.crop_size)

    def __call__(self, img1, img2, flow, params=None):
        """One sample -> (img1 (ch, cw, 3) uint8, img2, flow (ch, cw, 2) float32), as the reference's __call__."""
        out = self.batch([(img1, img2, flow)], None if params is None else [params])
        return out[0][0], out[1][0], out[2][0]


class SparseFlowAugmentor(_Augmentor):
    """Reference augmentor.py:132-267 on the GPU: symmetric colour with RandomBrightnessContrast(0.3, 0.3) and
    HueSaturationValue(17, 76, 0), the same eraser, a scale clipped to (crop + 1) / size without stretch, applied
    (p = 0.8) with cv2.resize to the images and resize_sparse_flow_map to the flow and valid, an h-flip (p = 0.5)
    when do_flip, and a crop drawn 20 rows / 50 columns beyond the image and clipped back."""
    _sparse = True
    _photo_limits = (0.3, (int(0.3 / 3.14 * 180), int(0.3 * 255), int(0.)))

    def __init__(self, crop_size, min_scale=-0.2, max_scale=0.5, do_flip=False, device='cuda'):
        super().__init__(crop_size, min_scale, max_scale, do_flip, device)

    def sample_params(self, ht, wd):
        colour = self._photo_params()                                    # :164
        rects = self._eraser_params(ht, wd)
        min_scale = np.maximum((self.crop_size[0] + 1) / float(ht), (self.crop_size[1] + 1) / float(wd))    # :221
        scale = 2 ** np.random.uniform(self.min_scale, self.max_scale)
        scale_x = np.clip(scale, min_scale, None)
        scale_y = np.clip(scale, min_scale, None)
        spatial = np.random.rand() < self.spatial_aug_prob
        hflip = False
        if self.do_flip:
            hflip = np.random.rand() < 0.5
        h1, w1 = (resized_size(ht, scale_y), resized_size(wd, scale_x)) if spatial else (ht, wd)
        y0 = np.random.randint(0, h1 - self.crop_size[0] + 20)           # :245
        x0 = np.random.randint(-50, w1 - self.crop_size[1] + 50)
        y0 = np.clip(y0, 0, h1 - self.crop_size[0])
        x0 = np.clip(x0, 0, w1 - self.crop_size[1])
        return AugmentParams(colour, colour, rects, float(scale_x), float(scale_y), bool(spatial), bool(hflip), False,
                             int(y0), int(x0), self.crop_size)

    def __call__(self, img1, img2, flow, valid, params=None):
        """One sample -> (img1, img2, flow, valid (ch, cw) float32), as the reference's __call__."""
        out = self.batch([(img1, img2, flow, valid)], None if params is None else [params])
        return tuple(t[0] for t in out)
