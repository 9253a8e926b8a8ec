#!/usr/bin/env python
"""Small end-to-end updates for compute-sanitizer (memcheck / racecheck / synccheck):
   compute-sanitizer --tool racecheck python tools/sanitize_case.py"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_configs import kwargs, sample
from gops_b200.create_pkg.create_alg import create_alg

torch.manual_seed(0)
which = sys.argv[1:] or ["idp", "lq", "veh", "wide", "tc", "lw", "dsac", "cstr", "detour", "peer"]
if "idp" in which:
    alg = create_alg(**kwargs("pyth_idpendulum", "FHADP", 6, 1, 64, "gelu", pre_horizon=3, reward_scale=1.0))
    for B in (700, 130):     # cfg1/cfg2 tiles incl. ragged tails
        alg.local_update(sample("pyth_idpendulum", B, 1), 0)
if "lq" in which:
    alg = create_alg(**kwargs("pyth_lq", "INFADP", 4, 2, 64, "relu", lq_config="s4a2", reward_scale=1.0))
    alg.set_parameters({"forward_step": 3})
    d = sample("pyth_lq", 300, 2)
    alg.local_update(d, 0)
    alg.local_update(d, 1)
if "veh" in which:
    alg = create_alg(**kwargs("pyth_veh3dofconti", "INFADP", 46, 2, 64, "relu", pre_horizon=10))
    alg.set_parameters({"forward_step": 2})
    d = sample("pyth_veh3dofconti", 200, 3, pre_horizon=10)
    alg.local_update(d, 0)
    alg.local_update(d, 1)
if "wide" in which:
    alg = create_alg(**kwargs("veh3dof_tracking", "FHADP", 46, 2, 256, "elu", pre_horizon=10))
    alg.set_parameters({"pre_horizon": 2})
    alg.local_update(sample("veh3dof_tracking", 70, 4, pre_horizon=10), 0)
if "tc" in which:          # wgmma kernels: tensor-core rollout (forced) and batched inference incl. a ragged tail
    os.environ["GOPS_B200_ROLLOUT"] = "tc"
    alg = create_alg(**kwargs("pyth_idpendulum", "FHADP", 6, 1, 64, "gelu", pre_horizon=3, reward_scale=1.0))
    for B in (700, 130):
        alg.local_update(sample("pyth_idpendulum", B, 1), 0)
    alg = create_alg(**kwargs("pyth_lq", "INFADP", 4, 2, 64, "relu", lq_config="s4a2", reward_scale=1.0))
    alg.set_parameters({"forward_step": 3})
    d = sample("pyth_lq", 300, 2)
    alg.local_update(d, 0)
    alg.local_update(d, 1)
    os.environ.pop("GOPS_B200_ROLLOUT")
    os.environ["GOPS_B200_INFER"] = "tc"
    alg.networks.policy(torch.randn(4321, 4, device="cuda"))
    alg.networks.v(torch.randn(129, 4, device="cuda"))
    os.environ.pop("GOPS_B200_INFER")
if "lw" in which:          # layer-wise wgmma path: wide FHADP (C3 shape, small), FHADP2, a bare LayerwiseMlp with ragged shapes
    alg = create_alg(**kwargs("veh3dof_tracking", "FHADP", 46, 2, 256, "elu", pre_horizon=10))
    alg.kernel_path = "tc"
    alg.set_parameters({"pre_horizon": 3})
    alg.local_update(sample("veh3dof_tracking", 200, 4, pre_horizon=10), 0)
    kw2 = kwargs("pyth_idpendulum", "FHADP2", 6, 1, 64, "gelu", pre_horizon=4, reward_scale=1.0)
    kw2["policy_func_name"] = "FiniteHorizonFullPolicy"
    alg = create_alg(**kw2)
    alg.local_update(sample("pyth_idpendulum", 333, 5), 0)
    from gops_b200.ops.layerwise_mlp import LayerwiseMlp
    net = LayerwiseMlp([19, 100, 37, 5], "tanh", max_batch=129)
    flat = torch.randn(net.nparam, device="cuda") * 0.1
    net.pack(flat)
    net.forward(torch.randn(129, 19, device="cuda"))
    g = torch.zeros(net.nparam, device="cuda")
    net.backward(torch.randn(129, 5, device="cuda"), grad=g, want_dx=True)
if "dsac" in which:
    kw3 = kwargs("pyth_idpendulum", "DSAC", 6, 1, 64, "gelu")
    kw3.update(policy_func_name="StochaPolicy", policy_hidden_sizes=[64, 64, 64], value_hidden_sizes=[64, 64, 64],
               policy_act_distribution="TanhGaussDistribution", policy_min_log_std=-20, policy_max_log_std=1,
               value_func_name="ActionValueDistri", alpha_learning_rate=1e-3, gamma=0.99, tau=0.005, auto_alpha=True,
               alpha=0.2, delay_update=2, TD_bound=10, bound=True)
    alg = create_alg(**kw3)
    B = 300
    d = {"obs": torch.randn(B, 6), "act": torch.rand(B, 1) * 2 - 1, "rew": torch.randn(B), "obs2": torch.randn(B, 6),
         "done": torch.zeros(B)}
    alg.local_update(d, 0)
    alg.local_update(d, 1)
if "cstr" in which:
    kw4 = kwargs("pyth_veh3dofconti_errcstr", "FHADPInterior", 46, 2, 64, "elu", pre_horizon=10, y_error_tol=1.2, u_error_tol=2.2)
    kw4["policy_func_name"] = "FiniteHorizonPolicy"
    alg = create_alg(**kw4)
    d = sample("pyth_veh3dofconti", 150, 6, pre_horizon=10)
    d["done"][::4] = 1.0
    alg.local_update(d, 0)
if "detour" in which:      # surrounding-vehicle model + interior point on the layer-wise path (lw_detour.cuh), done samples, ragged batch
    kw5 = kwargs("veh3dof_tracking_detour", "FHADPInterior", 50, 2, 64, "elu", pre_horizon=10, penalty=2.0)
    kw5["policy_func_name"] = "FiniteHorizonPolicy"
    alg = create_alg(**kw5)
    dd = sample("veh3dof_tracking_detour", 150, 7, pre_horizon=10)
    dd["done"][::4] = 1.0
    for i in range(3):       # eager, capture, replay
        alg.local_update(dd, i)
if "peer" in which:        # exchange + Adam kernel, single rank (the sanitizer serialises kernels: peers cannot spin on each other)
    from gops_b200.utils.peer_reduce import PeerReduce
    from gops_b200 import _lib
    import ctypes as C
    pr = PeerReduce(1, 0, 1000)
    buf, par, m, v = (torch.randn(777, device="cuda") for _ in range(4))
    v.abs_()
    _lib.check(_lib.lib().gops_b200_peer_allreduce(pr.handle, _lib.ptr(buf), 777, _lib.ptr(par), _lib.ptr(m), _lib.ptr(v), 773, 3,
                                                   1e-3, 0.9, 0.999, 1e-8, _lib.stream_ptr()))
    pr.allreduce(torch.randn(5, device="cuda"))
torch.cuda.synchronize()
print("sanitize_case done")
