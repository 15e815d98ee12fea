"""Host-side mirror of the reference's plugin interface for the BEV-encoder hot path
(projects/mmdet3d_plugin/bevformer/modules/__init__.py:3-5 exports the same names)."""
from .decoder import (CustomMSDeformableAttention, DetectionTransformerDecoder, DetrTransformerDecoderLayer,
                      GroupMultiheadAttention, MultiheadAttention, inverse_sigmoid)
from .encoder import FFN, BEVFormerEncoder, BEVFormerLayer, MyCustomBaseTransformerLayer
from .registry import (ATTENTION, FEEDFORWARD_NETWORK, TRANSFORMER_LAYER, TRANSFORMER_LAYER_SEQUENCE,
                       build_attention, build_from_cfg, build_transformer_layer,
                       build_transformer_layer_sequence)
from .spatial_cross_attention import MSDeformableAttention3D, ScaPlan, SpatialCrossAttention
from .temporal_self_attention import TemporalSelfAttention
from .temporal import BEVStream, obtain_history_bev
from .dcn import ModulatedDeformConv2d, ModulatedDeformConv2dPack
from .grid_mask import GridMask
from .head import BEVFormerHead, BEVFormerHead_GroupDETR, LearnedPositionalEncoding, NMSFreeCoder
from .registry import BBOX_CODERS, CONV_LAYERS, HEADS, POSITIONAL_ENCODING, build_conv_layer
from .transformer import (PerceptionTransformer, PerceptionTransformerBEVEncoder, PerceptionTransformerV2,
                          ResNetFusion)

__all__ = ["GridMask", "ModulatedDeformConv2d", "ModulatedDeformConv2dPack", "CONV_LAYERS", "build_conv_layer", "BEVFormerHead", "BEVFormerHead_GroupDETR", "LearnedPositionalEncoding", "NMSFreeCoder", "HEADS",
           "BBOX_CODERS", "POSITIONAL_ENCODING", "PerceptionTransformerV2", "ResNetFusion", "BEVStream", "obtain_history_bev", "PerceptionTransformer", "PerceptionTransformerBEVEncoder", "CustomMSDeformableAttention", "DetectionTransformerDecoder",
           "DetrTransformerDecoderLayer", "GroupMultiheadAttention", "MultiheadAttention", "inverse_sigmoid", "BEVFormerEncoder", "BEVFormerLayer", "MyCustomBaseTransformerLayer", "FFN",
           "SpatialCrossAttention", "MSDeformableAttention3D", "TemporalSelfAttention", "ScaPlan",
           "ATTENTION", "FEEDFORWARD_NETWORK", "TRANSFORMER_LAYER", "TRANSFORMER_LAYER_SEQUENCE",
           "build_attention", "build_from_cfg", "build_transformer_layer",
           "build_transformer_layer_sequence"]
