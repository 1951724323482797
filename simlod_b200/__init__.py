"""simlod_b200 — H100-native (sm_90a) implementation of SimLOD's two hot paths.

Only what the path needs lives here:
  csrc/       hand-written CUDA kernels (kernel_construct, kernel_render, reset `kernel`) and the
              C-ABI launch surface (include/simlod_b200.h)
  api.py      ctypes binding + `SimLOD`, the Python mirror of the reference host functions
              (resetCUDA / updateOctree / renderCUDA of main_progressive_octree.cpp)
  camera.py   OrbitControls / Camera / getUniforms restated (include/OrbitControls.h, GLRenderer.h)
  data.py     synthetic point streams of the benchmark configurations
  dist.py     batch sharding + reductions for one-process-per-GPU insertion
"""
from .api import SimLOD, SimlodError, make_points, POINT_DTYPE, load_library, read_las_header, Region, files_box  # noqa: F401
