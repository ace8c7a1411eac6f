"""reference path: upsnet/nms/nms.py -- gpu_nms_wrapper / py_nms_wrapper run the device-resident sm_90a NMS
(`IoU > thresh` suppresses, nms_kernel.cu:30-38 == py_nms nms.py:47-86).  cpu_nms_wrapper is NOT aliased: the reference's
Cython cpu_nms suppresses at `IoU >= thresh` (SURVEY F10), a different rule -- it raises instead of silently differing."""
from upsnet_b200.operators import gpu_nms, gpu_nms_wrapper  # noqa: F401


def py_nms_wrapper(thresh):
    """nms/nms.py:26-29; same `IoU > thresh` semantics as the GPU kernel, so it maps onto it."""
    return gpu_nms_wrapper(thresh, 0)


def cpu_nms_wrapper(thresh):
    raise NotImplementedError("cpu_nms (IoU >= thresh, nms/cpu_nms.pyx) has no sm_90a counterpart; use gpu_nms_wrapper "
                              "or py_nms_wrapper (IoU > thresh), the rule the hot path uses (mask_roi.py:40, pyramid_proposal.py:45)")
