"""flpr_b200 — a Hopper-native federated lifelong person-ReID engine.

Capabilities follow MSNLAB/Federated-Lifelong-Person-ReID (FedSTIL): ten federated / continual methods, ResNet and
Swin ReID backbones, CE / triplet / distillation criteria, CMC / mAP evaluation, accuracy / forgetting analysis,
the same YAML / log / checkpoint surfaces — re-designed for one 8xH100 node: one rank per GPU, flat device-resident
parameter arenas, NVLink peer-memory collectives and wgmma tensor-core kernels.
"""
__version__ = "0.1.0"
