"""H100-native (sm_90a) YOLOX hot path behind the yolov7_d2 registry surface."""
__version__ = "0.1.0"
