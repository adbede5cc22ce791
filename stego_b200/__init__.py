"""stego_b200 — H100-native (sm_90a) implementation of STEGO's feature-correspondence
distillation training step behind the reference's `modules.py` API surface."""

__version__ = "0.1.0"
