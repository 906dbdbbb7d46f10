"""humanvid_b200 -- Hopper-native (sm_90a) denoising path of CamAnimate / HumanVid.

Public surface mirrors the reference's modules for this path (see modules.py / pipeline.py); the arithmetic lives in
lib/libhv_b200.so, built by ``__graft_entry__.build()``.
"""
from .modules import (AutoencoderKL, BasicTransformerBlock, CameraPoseEncoder, CLIPVisionModelWithProjection, PoseGuider, ReferenceAttentionControl,
                      TemporalBasicTransformerBlock, UNet2DConditionModel, UNet2DConditionOutput, UNet3DConditionModel, UNet3DConditionOutput)
from .scheduler import DDIMScheduler
from . import camera

__all__ = ["UNet3DConditionModel", "UNet3DConditionOutput", "UNet2DConditionModel", "UNet2DConditionOutput", "PoseGuider", "CameraPoseEncoder",
           "ReferenceAttentionControl", "TemporalBasicTransformerBlock", "BasicTransformerBlock", "DDIMScheduler", "AutoencoderKL",
           "CLIPVisionModelWithProjection"]
