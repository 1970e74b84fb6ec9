"""occformer_b200 -- H100 (sm_90a) native hot path of OccFormer behind the reference's plugin surface.

Registry names / constructor kwargs / forward signatures / state_dict keys follow
projects/mmdet3d_plugin of the reference; all arithmetic runs in csrc/libocc_b200.so (C ABI, ctypes).
"""
from .registry import ATTENTION, BACKBONES, DETECTORS, HEADS, NECKS, PIPELINES, POSITIONAL_ENCODING  # noqa: F401
from .encoder import DualpathTransformerBlock, OccupancyEncoder  # noqa: F401
from .image_encoder import SECONDFPN, ResNet, ResNetDCN  # noqa: F401
from .efficientnet import CustomEfficientNet  # noqa: F401
from .view_transformer import ViewTransformerLiftSplatShootVoxel, bev_pool  # noqa: F401
from .neck import MSDeformAttnPixelDecoder3D, MultiScaleDeformableAttention3D  # noqa: F401
from .head import (Mask2FormerNuscOccHead, Mask2FormerNuscPanopticOccHead, Mask2FormerOccHead,  # noqa: F401
                   SinePositionalEncoding3D)
from .detector import OccupancyFormer  # noqa: F401
from .pipelines import (LoadMultiViewImageFrames_OccFormer, LoadMultiViewImageFrames_SemanticKitti,  # noqa: F401
                        LoadMultiViewJpegBytes_OccFormer, LoadMultiViewPngBytes_SemanticKitti,
                        LoadNuscOccupancyPoints, LoadNuscPanopticOccupancyPoints, LoadSemKittiVoxelFiles)

__version__ = "0.1.0"
