"""micro_sam_b200 -- the SAM hot path of micro-sam (embedding precompute, prompt decode, AMG post-processing) as
hand-written sm_90a CUDA behind a C ABI (include/msam_b200.h), exposed through micro-sam's own function signatures."""
__version__ = "0.2.0"
