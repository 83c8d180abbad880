"""The reference's data pipeline: file formats (tf_raft/datasets/frame_utils.py: Middlebury .flo and KITTI flow PNGs)
and the training augmentors (tf_raft/datasets/augmentor.py) on the GPU."""
from .augmentor import AugmentParams, FlowAugmentor, SparseFlowAugmentor  # noqa: F401
from .frame_utils import read_flow, read_flow_kitti, write_flow, write_flow_kitti  # noqa: F401
