"""vlp_b200 — H100-native (sm_90a) implementation of LuoweiZhou/VLP's data-parallel hot path.

Python keeps the reference's nn.Module surface (vlp_b200.vlp_modules); all device work is done by
hand-written CUDA in libvlpk.so behind a C ABI (include/vlpk.h).
"""
__version__ = "0.1.0"
