"""The reference's data pipeline: the datasets (tf_raft/datasets/dataset.py) with a batch loader, file formats
(tf_raft/datasets/frame_utils.py: Middlebury .flo, PFM, KITTI flow PNGs, the latter also decoded on the GPU), the
training augmentors (tf_raft/datasets/augmentor.py) and the flow colour wheel (tf_raft/datasets/flow_viz.py) on the
GPU."""
from .augmentor import AugmentParams, FlowAugmentor, SparseFlowAugmentor  # noqa: F401
from .dataset import HD1K, KITTI, FlowDataset, FlyingChairs, FlyingThings3D, MpiSintel, as_supervised  # noqa: F401
from .flow_viz import flow_to_image, flow_uv_to_colors, make_colorwheel  # noqa: F401
from .frame_utils import (inflate_png16, read_flow, read_flow_kitti, read_gen, read_pfm, write_flow,  # noqa: F401
                          write_flow_kitti, write_png)
from .png16 import decode_png16, read_flow_kitti_batch  # noqa: F401
from ..preprocess import CropOrPadder  # noqa: F401
