"""The reference's data pipeline: file formats (tf_raft/datasets/frame_utils.py: Middlebury .flo and KITTI flow PNGs),
the training augmentors (tf_raft/datasets/augmentor.py) and the flow colour wheel (tf_raft/datasets/flow_viz.py) on the
GPU."""
from .augmentor import AugmentParams, FlowAugmentor, SparseFlowAugmentor  # noqa: F401
from .flow_viz import flow_to_image, flow_uv_to_colors, make_colorwheel  # noqa: F401
from .frame_utils import read_flow, read_flow_kitti, write_flow, write_flow_kitti, write_png  # noqa: F401
