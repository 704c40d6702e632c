"""stylesinger_b200 — H100-native (sm_90a) engine for StyleSinger's ph -> mel -> wav hot path.

Host side (this package): tensor plumbing, checkpoint packing, the drop-in mirrors of the
reference's Python interfaces.  All arithmetic of the hot path runs in hand-written CUDA kernels
behind the C ABI declared in include/stylesinger_b200.h (stylesinger_b200/csrc).  There is no CPU
or PyTorch fallback: importing the compute entry points without the built library raises.
"""
__version__ = "0.1.0"
