"""The DeMoN v2 network (python/depthmotionnet/v2): `networks` (BootstrapNet, IterativeNet, RefinementNet,
DemonPipelineV2) and `weights` (its variable table)."""
