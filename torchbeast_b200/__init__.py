"""torchbeast_b200: H100-native (sm_90a) IMPALA learner hot path behind torchbeast's API.

Python surface mirrors the reference (facebookresearch/torchbeast):
    torchbeast_b200.core.vtrace        <- torchbeast/core/vtrace.py
    torchbeast_b200.monobeast          <- torchbeast/monobeast.py   (learn, AtariNet, compute_*_loss)
    torchbeast_b200.polybeast_learner  <- torchbeast/polybeast_learner.py (learn, Net, compute_*_loss)
All device work goes through the C-ABI library declared in include/torchbeast_b200.h.
"""
__version__ = "0.1.0"
