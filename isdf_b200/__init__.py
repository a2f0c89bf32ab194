"""isdf_b200 -- H100 (sm_90a) implementation of the iSDF continual-training hot path.

Host side mirrors the reference's Python interface (isdf.modules.trainer.Trainer and
isdf.modules.{fc_map,embedding,sample,loss,render}); compute goes through the C ABI in
include/isdf_b200.h (isdf_b200/lib/libisdf_b200.so, built by __graft_entry__.build()).
"""
__version__ = "0.1.0"

DEFAULT_PRECISION = "bf16x3g"    # overridden by env ISDFB_PRECISION or the config's "b200" section
