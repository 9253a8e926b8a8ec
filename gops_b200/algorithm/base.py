"""Algorithm / approximate-function-container base classes (reference: gops/algorithm/base.py:24-120),
plus the shared plumbing of the fused ADP algorithms: plan creation, batch marshalling, the single
NCCL all-reduce of the flat gradient, and the fused Adam step."""
import ctypes as C
from abc import ABC, ABCMeta, abstractmethod
from copy import deepcopy
from typing import Dict, Optional, Tuple

import torch

from gops_b200 import _lib
from gops_b200.create_pkg.create_apprfunc import create_apprfunc
from gops_b200.env.fused import fill_plan_desc, make_batch
from gops_b200.utils.common_utils import get_apprfunc_dict, set_seed
from gops_b200.utils.flat_params import GRAD_TAIL, FlatParams


class ApprBase(ABC, torch.nn.Module):
    """Base class of approximate-function containers."""

    def __init__(self, **kwargs):
        super().__init__()
        if kwargs.get("cnn_shared"):
            raise NotImplementedError("gops_b200: cnn_shared feature networks are outside the MLP hot path")

    def init_scheduler(self, **kwargs):
        assert hasattr(self, "optimizer_dict")
        self.scheduler_dict = {}
        for key in [k for k in kwargs if k.endswith("_scheduler")]:
            self.scheduler_dict[key] = getattr(torch.optim.lr_scheduler, kwargs[key]["name"])(
                self.optimizer_dict[key.replace("_scheduler", "")], **kwargs[key]["params"])


def target_copy(net: torch.nn.Module) -> torch.nn.Module:
    """A Polyak target of `net`: a deep copy whose parameters take no gradient.  Made before the first update, the copy
    owns its own `FlatParams` (bound to the copied module) and library handles."""
    target = deepcopy(net)
    for p in target.parameters():
        p.requires_grad = False
    return target


class AlgorithmBase(metaclass=ABCMeta):
    """Base class of algorithms: same surface as the reference (local_update / get_remote_update_info /
    remote_update / state_dict / set_parameters ...)."""

    def __init__(self, index, **kwargs):
        self.networks = None
        set_seed(kwargs["trainer"], kwargs["seed"], index + 300)

    @property
    @abstractmethod
    def adjustable_parameters(self) -> tuple:
        ...

    def set_parameters(self, param_dict):
        for key in param_dict:
            if hasattr(self, key) and key in self.adjustable_parameters:
                setattr(self, key, param_dict[key])
            else:
                raise RuntimeError("param '" + key + "'is not adjustable in algorithm!")

    def get_parameters(self):
        return dict(zip(self.adjustable_parameters, (getattr(self, p) for p in self.adjustable_parameters)))

    def state_dict(self):
        return self.networks.state_dict()

    def load_state_dict(self, state_dict):
        self.networks.load_state_dict(state_dict)

    def local_update(self, data: dict, iteration: int) -> dict:
        tb_info = self._local_update(data, iteration)
        for scheduler in self.networks.scheduler_dict.values():
            scheduler.step()
        return tb_info

    def remote_update(self, update_info: dict):
        self._remote_update(update_info)
        for scheduler in self.networks.scheduler_dict.values():
            scheduler.step()

    def _local_update(self, data: dict, iteration: int) -> dict:
        pass

    def get_remote_update_info(self, data: dict, iteration: int) -> Tuple[dict, dict]:
        raise NotImplementedError

    def _remote_update(self, update_info: dict):
        raise NotImplementedError

    def to(self, device):
        self.networks.to(device)

    def _device(self) -> torch.device:
        """The networks' device; networks still on the CPU are moved to CUDA first (the updates run there only)."""
        p = next(self.networks.parameters())
        if not p.is_cuda:
            if not torch.cuda.is_available():
                raise RuntimeError(f"gops_b200: no CUDA device -- the {type(self).__name__} update has no CPU fallback")
            self.networks.cuda()
            p = next(self.networks.parameters())
        return p.device

    def train(self):
        self.networks.train()

    def eval(self):
        self.networks.eval()


class RolloutPlan:
    """Owns one `gops_b200_plan` (C side) for a fixed (algorithm kind, horizon, gamma, env, nets)."""

    def __init__(self, alg_kind: int, envmodel, policy, value, horizon: int, gamma: float, device=None,
                 open_loop: bool = False):
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(self.device):     # the C side allocates its scratch on the current device
            self._create(alg_kind, envmodel, policy, value, horizon, gamma, open_loop)

    def _create(self, alg_kind, envmodel, policy, value, horizon, gamma, open_loop):
        desc = _lib.PlanDesc()
        desc.open_loop = int(open_loop)
        desc.alg, desc.horizon, desc.gamma = alg_kind, int(horizon), float(gamma)
        desc.policy = policy.mlp_desc()
        if value is not None:
            desc.value = value.mlp_desc()
        keep = fill_plan_desc(desc, envmodel, policy.act_low_lim.detach().cpu().numpy(),   # noqa: F841 (keeps arrays alive)
                              policy.act_high_lim.detach().cpu().numpy())
        self.handle = C.c_void_p()
        _lib.check(_lib.lib().gops_b200_plan_create(C.byref(desc), C.byref(self.handle)))
        _lib.check(_lib.lib().gops_b200_plan_set_gamma(self.handle, float(gamma)))
        self.gamma = float(gamma)
        self.key = (alg_kind, int(horizon))

    def set_gamma(self, gamma: float):
        if float(gamma) != self.gamma:
            _lib.check(_lib.lib().gops_b200_plan_set_gamma(self.handle, float(gamma)))
            self.gamma = float(gamma)

    def set_path(self, path: str):
        """'auto' | 'mma' | 'tc': kernel path of the fused rollout (raises if 'tc' is not built for this plan)."""
        _lib.check(_lib.lib().gops_b200_plan_set_path(
            self.handle, {"auto": _lib.PATH_AUTO, "mma": _lib.PATH_MMA, "tc": _lib.PATH_TC}[path]))

    def last_path(self) -> str:
        """Kernel path the most recent rollout launch of this plan took ('none' before the first launch)."""
        return _lib.PATH_NAMES[_lib.lib().gops_b200_plan_last_path(self.handle)]

    def __del__(self):
        try:
            if self.handle:
                _lib.lib().gops_b200_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


def shard_inv_batch(local_batch: int, world: int) -> float:
    """1 / B_global for equal shards: every rank scales its partial loss/gradient sums by this, so that the
    SUM all-reduce yields the global batch mean -- the semantics of the reference's OffSyncTrainer, which
    averages the replicas' gradients (gops/trainer/off_sync_trainer.py:183-208)."""
    return 1.0 / float(local_batch * world)


def allreduce_flat(gbuf: torch.Tensor, optimizer=None) -> bool:
    """ONE exchange per optimizer step over [flat gradient | loss | critic mean | #done].  Between GPUs of one node it
    is a single kernel over NVLink peer memory (utils/peer_reduce.py) which also applies `optimizer`'s Adam step;
    otherwise an NCCL / gloo all-reduce.  Returns True when the optimizer step has been applied here."""
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        if gbuf.is_cuda:
            from gops_b200.utils.peer_reduce import group_peer
            peer = group_peer(gbuf.numel(), gbuf.device)
            if peer is not None:
                peer.allreduce(gbuf, optimizer)
                return optimizer is not None
        dist.all_reduce(gbuf, op=dist.ReduceOp.SUM)
    return False


class FusedADPMixin:
    """Shared by FHADP / INFADP: plans cache, fused rollout-gradient call."""

    def _init_fused(self):
        self._plans: Dict[tuple, RolloutPlan] = {}
        if torch.cuda.is_available():
            self.networks.cuda()

    kernel_path = "auto"     # 'auto' | 'mma' | 'tc' (RolloutPlan.set_path); tests state and assert the path here
    MAX_PLANS = 4            # LRU: annealing pre_horizon must not leak one tape + blobs per distinct value

    def _plan(self, alg_kind, policy, value, horizon, gamma, open_loop: bool = False) -> RolloutPlan:
        dev = self._device()
        key = (alg_kind, int(horizon), dev.index)
        plan = self._plans.pop(key, None)
        if plan is None:
            plan = RolloutPlan(alg_kind, self.envmodel, policy, value, horizon, gamma, device=dev, open_loop=open_loop)
            while len(self._plans) >= self.MAX_PLANS:
                self._plans.pop(next(iter(self._plans)))          # least recently used; its __del__ frees the C plan
        self._plans[key] = plan                                   # most recently used last
        plan.set_gamma(gamma)                                     # gamma is a table in the plan, not a new plan
        if plan.__dict__.get("_path") != self.kernel_path:
            plan.set_path(self.kernel_path)
            plan._path = self.kernel_path
        return plan

    # ---- loss read-back -------------------------------------------------------------------------------------------
    # The reference reads `loss.item()` inside _compute_gradient, i.e. BEFORE the optimizer step is launched; here that
    # would idle the GPU between the rollout and Adam.  The 4-float tail [loss | v-mean | #done | pad] is instead copied
    # to pinned host memory AFTER the optimizer launches of the step:
    #   loss_lag = 0 (default): wait for this step's copy -> tb_info carries this step's loss (reference semantics);
    #   loss_lag = 1: tb_info carries the PREVIOUS step's loss (this step's on the first call), so the host runs one
    #                 step ahead of the device and no launch gap is exposed (bench.py states which mode it times).
    loss_lag = 0

    def _tail_to_host(self, *tails: torch.Tensor):
        """The device tails of one update, side by side in one pinned buffer, as a host list (honours loss_lag)."""
        ring = self.__dict__.get("_tail_ring")
        if ring is None:
            ring = [(torch.zeros(len(tails) * GRAD_TAIL, dtype=torch.float32).pin_memory(), torch.cuda.Event())
                    for _ in range(2)]
            self.__dict__["_tail_ring"] = ring
            self.__dict__["_tail_n"] = 0
        n = self.__dict__["_tail_n"]
        buf, ev = ring[n % 2]
        with torch.cuda.device(tails[0].device):
            for i, tail in enumerate(tails):
                buf[i * GRAD_TAIL:(i + 1) * GRAD_TAIL].copy_(tail, non_blocking=True)
            ev.record()
        self.__dict__["_tail_n"] = n + 1
        if self.loss_lag and n > 0:
            buf, ev = ring[(n - 1) % 2]
        ev.synchronize()
        return buf.tolist()

    def last_kernel_path(self) -> str:
        """Path of the most recent fused rollout launch ('mma' | 'tc'), for tests and bench bookkeeping."""
        return next(reversed(self._plans.values())).last_path() if self._plans else "none"

    @staticmethod
    def _world():
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            return dist, dist.get_world_size()
        return None, 1

    def _launch_and_step(self, launch, optimizer):
        """`launch()` (a fused rollout-gradient call) followed by `optimizer.step()`.  On several GPUs the step is
        applied inside the gradient-exchange kernel instead of by a launch of its own."""
        self._fuse_opt, self._opt_applied = optimizer, False
        try:
            out = launch()
        finally:
            self._fuse_opt = None
        if not self._opt_applied:
            optimizer.step()
        return out

    def _rollout_grad(self, plan: RolloutPlan, data: dict, target: FlatParams, policy: FlatParams,
                      value: Optional[FlatParams], vtarget: Optional[FlatParams]) -> torch.Tensor:
        """Runs the fused kernel on this rank's shard and all-reduces [grad | loss | v-mean | #done].
        Returns the 4-float tail as a device tensor (no host sync here)."""
        dev = self._device()
        base = self.envmodel.unwrapped
        obs = data["obs"]
        obs_d = obs.to(dev, non_blocking=True) if not obs.is_cuda else obs
        done = data["done"]
        done_d = done.to(dev, non_blocking=True) if not done.is_cuda else done
        dist, world = self._world()
        B_local = obs_d.shape[0]
        inv_B = shard_inv_batch(B_local, world)
        target.bind_grads()
        gbuf = target.gbuf
        n = gbuf.numel() - GRAD_TAIL
        keep = []
        with torch.cuda.device(dev):
            info = {k: (v.to(dev, non_blocking=True) if torch.is_tensor(v) and not v.is_cuda else v)
                    for k, v in data.items() if k not in ("obs", "done")}
            batch = make_batch(base, obs_d, done_d, info, keep)
            _lib.check(_lib.lib().gops_b200_rollout_grad(
                plan.handle, C.byref(batch), _lib.ptr(policy.sync()),
                _lib.ptr(value.sync()) if value is not None else None,
                _lib.ptr(vtarget.sync()) if vtarget is not None else None,
                C.c_float(inv_B), _lib.ptr(gbuf), C.c_void_p(gbuf.data_ptr() + 4 * n), _lib.stream_ptr()))
            opt, self._fuse_opt = getattr(self, "_fuse_opt", None), None
            self._opt_applied = allreduce_flat(gbuf, opt)
        return gbuf[n:]
