"""fast3r_b200 — H100-native (sm_90a) implementation of the Fast3R single-forward-pass hot path.

Public surface mirrors the reference: ``Fast3R`` (fast3r/models/fast3r.py:45) and ``inference`` /
``loss_of_one_batch`` (fast3r/dust3r/inference_multiview.py).  The compute lives in ``libfast3r_b200.so``
(hand-written CUDA, C ABI in include/fast3r_b200.h)."""
from .model import Fast3R  # noqa: F401
from .inference import inference, inference_many, loss_of_one_batch  # noqa: F401
from .configs import vit_large_args, tiny_args  # noqa: F401
