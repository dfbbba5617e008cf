"""b200seg — Hopper-native (sm_90a) training hot path for the 3D segmentation models of
yhygao/CBIM-Medical-Image-Segmentation, behind the reference's own interfaces:
``get_model(args)`` (model/utils.py:6), the module/state_dict contract, ``DiceLoss`` (training/losses.py:8).
Importing this package never touches the GPU; every op fails loudly without libb200seg.so + an H100."""
from . import _lib
from . import augmentation
from ._lib import B200SegError, EXPORTED_SYMBOLS, LIB_PATH
from .attention_unet import AttentionUNet
from .factory import get_model
from .inference import (calculate_dice, calculate_dice_split, calculate_distance, get_inference, inference_sliding_window,
                        inference_sliding_window_2d, inference_whole_image, inference_whole_image_2d)
from .losses import CrossEntropyLoss, DiceCELoss, DiceLoss
from .medformer import MedFormer
from .swin_unetr import SwinUNETR
from .unet2d import UNet2D
from .unet3d import UNet
from .unetpp import UNetPlusPlus
from .unetr import UNETR

__all__ = ["augmentation", "get_model", "UNet", "UNet2D", "MedFormer", "SwinUNETR", "UNETR", "UNetPlusPlus", "AttentionUNet", "DiceLoss", "DiceCELoss", "CrossEntropyLoss", "B200SegError",
           "EXPORTED_SYMBOLS", "LIB_PATH", "get_inference", "inference_sliding_window", "inference_whole_image", "inference_sliding_window_2d",
           "inference_whole_image_2d",
           "calculate_dice", "calculate_dice_split", "calculate_distance"]
