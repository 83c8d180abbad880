"""tf_raft_b200 -- H100-native (sm_90a) RAFT forward/update hot path behind the Python API of
daigo0927/tf-raft: `CorrBlock`, `BasicUpdateBlock` / `SmallUpdateBlock`, `RAFT` / `SmallRAFT`.

Compute lives in libraft_b200.so (hand-written CUDA, C ABI in include/raft_b200.h); PyTorch supplies
device memory, streams, CUDA graphs and torch.distributed.  No CPU fallback.
"""
from . import _lib
from .layers.corr import (CorrBlock, bilinear_sampler, coords_grid, fb_occlusion, forward_interpolate, tfa_sampler,
                          upflow8)
from .layers.extractor import BasicEncoder, SmallEncoder
from .layers.update import BasicUpdateBlock, SmallUpdateBlock
from .losses import EndPointError, UnsupervisedLoss, end_point_error, sequence_loss
from .model import RAFT, SmallRAFT
from .warp import compose_flow, warp
from .checkpoint import (load_pytorch_checkpoint, load_tf_checkpoint, param_to_tf_key, read_tf_checkpoint, tf_key_to_param,
                         to_pytorch_state_dict, write_tf_checkpoint)
from .preprocess import CropOrPadder, InputPadder, pad_to_multiple, resize_with_crop_or_pad
from .fit import Callback, History
from .train import (AdamW, CyclicalLearningRate, ModelCheckpoint, OneCycleLR, TensorBoard, TorchAdamW, VisFlowCallback,
                    first_cycle_scaler, inverse_scaler)
from .evaluation import FlowMetrics, evaluate, flow_metrics
from . import datasets
from .submission import create_kitti_submission, create_sintel_submission

__all__ = ['CorrBlock', 'bilinear_sampler', 'coords_grid', 'fb_occlusion', 'forward_interpolate', 'tfa_sampler', 'upflow8',
           'warp', 'compose_flow', 'BasicEncoder', 'SmallEncoder',
           'BasicUpdateBlock', 'SmallUpdateBlock', 'RAFT', 'SmallRAFT', 'sequence_loss', 'end_point_error', 'UnsupervisedLoss',
           'resize_with_crop_or_pad', 'CropOrPadder', 'InputPadder', 'pad_to_multiple',
           'load_pytorch_checkpoint', 'load_tf_checkpoint', 'to_pytorch_state_dict', 'TorchAdamW', 'OneCycleLR',
           'read_tf_checkpoint', 'write_tf_checkpoint', 'param_to_tf_key', 'tf_key_to_param', 'FlowMetrics', 'evaluate', 'flow_metrics',
           'Callback', 'History', 'ModelCheckpoint', 'TensorBoard', 'create_sintel_submission',
           'create_kitti_submission']
