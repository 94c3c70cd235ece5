"""yolov5_b200 -- H100-native (sm_90a) engine for the YOLOv5 forward / NMS / loss hot path.

Public surface mirrors the reference's Python callables for that path:
    yolov5_b200.models.yolo.DetectionModel / SegmentationModel / Detect / Segment / parse_model
    yolov5_b200.models.common.Conv / Bottleneck / C3 / SPPF / Concat / Proto
    yolov5_b200.utils.general.non_max_suppression, xywh2xyxy, ...
    yolov5_b200.utils.metrics.box_iou
    yolov5_b200.utils.loss.ComputeLoss
All arithmetic runs in liby5b200.so (hand-written CUDA behind the C ABI of include/y5b200.h).
"""
__version__ = "0.1.0"
