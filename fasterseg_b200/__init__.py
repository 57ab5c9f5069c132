"""fasterseg_b200 -- H100-native (sm_90a) implementation of the FasterSeg conv hot path behind the
reference's own operator API (operations / slimmable_ops / seg_oprs / model_seg / model_search)."""
__version__ = "0.1.0"
