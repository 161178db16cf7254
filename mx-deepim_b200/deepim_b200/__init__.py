"""deepim_b200 -- H100-native (sm_90a) render-and-compare pose refinement hot path of mx-DeepIM.

Python host over the C ABI in include/deepim_b200.h.  The names mirror the reference:
  deepim_b200.operator_py.*      <- deepim/operator_py/*.py   (ZoomMask, ZoomImageWithFactor, ...)
  deepim_b200.render_py_multi    <- lib/render_glumpy/render_py_multi.py (Render_Py)
  deepim_b200.RT_transform       <- lib/pair_matching/RT_transform.py (RT_transform)
  deepim_b200.gpu_flow           <- lib/flow_c/gpu_flow.pyx (gpu_flow)
  deepim_b200.refiner            <- the 4-iteration loop of deepim/core/tester.py:340-485
There is no CPU fallback: importing the op modules without libdeepim_b200.so raises.
"""
__version__ = "0.1.0"
