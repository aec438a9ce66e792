"""lav_b200 — H100-native (sm_90a) kernels and drop-in mirrors for the LAV frame path.

Layers: ``include/lav_b200.h`` (C ABI) -> ``csrc/*.cu`` built by ``lav_b200.build`` into ``_lib/liblavb200.so`` ->
``capi`` (ctypes) -> ``ops`` (tensor front ends) -> mirrors of the reference modules (``erfnet``, ``rgb``, ``point_painting``,
``point_pillar``, ``lidar``, ``heads``, ``model_inference``, ``agent``, ``train``).  There is no CPU fallback.
"""
__version__ = "0.1.0"
