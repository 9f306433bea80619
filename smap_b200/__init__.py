"""smap_b200 - H100-native (sm_90a) implementation of the SMAP inference hot path:
backbone forward + depth-aware part association + 3D lift, behind a C ABI (include/smap_b200.h).

There is no CPU or PyTorch fallback: importing `smap_b200.engine` loads libsmap_b200.so and every
operation fails loudly if the library or an H100 is missing."""
__version__ = "0.1.0"
