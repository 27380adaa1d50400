"""Host-side mirror of the reference's ``lib`` package for the inference hot path (H100 native).

Same module / function / class names as tsurumeso/vocal-remover's ``lib`` (nets, spec_utils, dataset),
backed by the hand-written sm_90a CUDA library ``libvr_b200.so`` through a C ABI (include/vr_b200.h).
Python/PyTorch here only loads weights, owns device buffers and orchestrates.
"""
