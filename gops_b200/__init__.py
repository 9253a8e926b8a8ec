"""gops_b200: H100-native (sm_90a CUDA) implementation of GOPS's batched model-rollout +
ADP-update hot path behind GOPS's own plugin API.

Layout mirrors the reference package for the modules on the path:
  gops_b200.create_pkg.{create_env_model, create_apprfunc, create_alg}
  gops_b200.algorithm.{base, fhadp, infadp}
  gops_b200.apprfunc.mlp
  gops_b200.env.env_ocp.env_model.{pyth_idpendulum_model, pyth_lq_model, pyth_veh3dofconti_model}
  gops_b200.env.env_gen_ocp.env_model.veh3dof_tracking_model
  gops_b200.env.wrapper.*
All arithmetic of the path runs in libgops_b200.so (gops_b200/csrc); there is no CPU fallback.
"""
__version__ = "0.1.0"
