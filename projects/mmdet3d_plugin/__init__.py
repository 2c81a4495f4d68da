"""Drop-in plug-in package for the DeepInteraction MMRI+MMPI forward path on H100 (libdi_b200, sm_90a).

Same import path and registered class names as the reference's ``projects/mmdet3d_plugin`` for the hot
path, so ``plugin=True; plugin_dir='projects/mmdet3d_plugin/'`` in Fusion_0075_*.py resolves
``type='DeepInteractionEncoder'`` / ``type='DeepInteractionDecoder'`` / ``type='TransFusionBBoxCoder'`` and, for
Fusion_0075_plusplus.py, ``type='FusionTransformerv4'`` (+ ``DeepInteractionLayer``, ``MMRI_P2I``, ``MMRI_I2P``,
``MMRI_I2P_Polar``) and ``type='DeepInteractionPlusPlusDecoder'`` to the libdi_b200-backed modules.  Everything outside the hot path (detector wrapper, backbones, data
pipelines, assigners, hooks) is out of scope (SURVEY.md section 8) and stays with the reference package.
"""
from .models.dense_heads.deepinteraction_decoder import DeepInteractionDecoder  # noqa: F401
from .models.dense_heads.deepinteractionplusplus_decoder import DeepInteractionPlusPlusDecoder  # noqa: F401
from .models.necks.deepinteraction_encoder import DeepInteractionEncoder  # noqa: F401
from .models.necks.fusion_transformerv4 import (FusionTransformerv4, DeepInteractionLayer, MMRI_P2I, MMRI_I2P,  # noqa: F401
                                                MMRI_I2P_Polar)
from .core.bbox.coders.transfusion_bbox_coder import TransFusionBBoxCoder  # noqa: F401
from .core.bbox.assigners.hungarian_assigner import (HungarianAssigner3D, HeuristicAssigner3D, BBox3DL1Cost,  # noqa: F401
                                                     BBoxBEVL1Cost, IoU3DCost)
