"""multiyolov5_b200 - H100-native (sm_90a) implementation of the joint detection+segmentation hot path of
TomMao23/multiyolov5 behind the reference's own Python surface:

    from multiyolov5_b200.models.yolo import Model              # reference models/yolo.py:233
    from multiyolov5_b200.utils.general import non_max_suppression, seg_argmax   # reference utils/general.py:421

All device work runs in libmyolo_sm90a.so (hand-written CUDA, C ABI in include/myolo.h); PyTorch only provides
tensors, streams and torch.distributed.
"""
__version__ = "0.1.0"
