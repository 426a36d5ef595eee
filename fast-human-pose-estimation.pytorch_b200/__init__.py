"""fpd_b200 -- H100 (sm_90a) native hot path for ilovepose/fast-human-pose-estimation.pytorch.

Import name: `fpd_b200` (the directory keeps the task-mandated name
`fast-human-pose-estimation.pytorch_b200/`, which is not a Python identifier; the repo-root shim
`fpd_b200.py` maps one onto the other).
"""
__version__ = "0.1.0"
