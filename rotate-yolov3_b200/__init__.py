"""H100-native hot path of ming71/rotate-yolov3 behind the reference's own Python signatures.

    from rotate_yolov3_b200 import r_nms, non_max_suppression, skew_bbox_iou, Darknet

All compute runs in ``libryolo.so`` (hand-written sm_90a CUDA behind the C-ABI of ``include/ryolo.h``);
importing the package fails loudly when that library has not been built -- there is no CPU fallback."""
from . import _lib  # noqa: F401  (raises ImportError with the build instruction if libryolo.so is missing)
from .iou import rotated_iou_matrix, skew_bbox_iou  # noqa: F401
from .nms import detect_multiscale, multiscale_sizes, nms_filter, non_max_suppression, r_nms  # noqa: F401
from .models import Darknet, YOLOLayer  # noqa: F401
from .preprocess import letterbox, letterbox_labels, scale_coords  # noqa: F401
from .augment import train_batch  # noqa: F401
from .decode import decode_images  # noqa: F401

__all__ = ["r_nms", "non_max_suppression", "nms_filter", "skew_bbox_iou", "rotated_iou_matrix", "Darknet", "YOLOLayer",
           "letterbox", "letterbox_labels", "scale_coords", "train_batch", "decode_images", "detect_multiscale",
           "multiscale_sizes"]
