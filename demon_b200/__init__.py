"""demon_b200 -- H100-native (sm_90a) DeMoN two-view depth+motion inference path.

  demon_b200.lmbspecialops       mirror of the reference op binding (warp2d, depth_to_flow, ...)
  demon_b200.networks_original   mirror of depthmotionnet.networks_original (BootstrapNet, ...)
  demon_b200.weights             TF variable table + seeded synthetic weights
  demon_b200.sequence            a video into one chained trajectory, a dense or sparse TSDF volume and its mesh
  demon_b200.mesh                connected components of an indexed mesh, and the mesh without its small ones
  demon_b200.build               nvcc build of libdemon_b200.so (C ABI in include/demon_b200.h)
"""
__version__ = "0.1"
