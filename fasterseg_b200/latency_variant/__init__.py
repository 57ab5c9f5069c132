"""The reference's latency/ deployment network (nearest resizes, single-conv stride-2 FactorizedReduce), inference only.
`zoo.build_network(..., variant="latency")` builds it; `python -m fasterseg_b200.launch` shadows `operations` / `model_seg` with
these modules for scripts in a directory named `latency`."""
