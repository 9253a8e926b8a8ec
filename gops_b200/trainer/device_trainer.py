"""On-device serial trainer: the caller of the fused ADP update (SURVEY.md 8(f) N2).

The reference's serial loop (gops/trainer/off_serial_trainer.py:79-173) steps a NumPy data env on the CPU, fills a
host replay buffer and copies a batch to the GPU for every update.  For the model-based ADP algorithms the replay
batch only provides INITIAL STATES, so here they are drawn directly on the device from the data envs' initial-state
distributions (idpendulum: pyth_idpendulum.py:36-38 uniform box; LQ: lq_base.py:151-155 Gaussian init_mean/init_std)
and handed to `alg.local_update` without any host round trip.  TensorBoard tags, the `apprfunc_{it}.pkl` checkpoint
format and the `config.json` dump follow the reference so that `example_run/*` keeps working on the results."""
import json
import os
import time
from typing import Dict, Optional

import torch

from gops_b200.utils.tensorboard_setup import tb_tags


class DeviceStateSampler:
    """Batched initial-state sampler living on the GPU (plumbing: torch RNG, no arithmetic of the hot path); the laws
    are the data envs' reset distributions, see gops_b200/trainer/device_sampler.py."""

    def __init__(self, env_id: str, device, seed: int = 0, **kwargs):
        from gops_b200.trainer import device_sampler as ds
        self.env_id, self.device = env_id, torch.device(device)
        self.gen = torch.Generator(device=self.device).manual_seed(int(seed))
        P = kwargs.get("pre_horizon", 10)
        if env_id == "pyth_idpendulum":
            self._draw = lambda b: ds.sample_idpendulum(b, self.device, gen=self.gen)
        elif env_id == "pyth_lq":
            cfg = kwargs.get("lq_config", "s3a1")
            self._draw = lambda b: ds.sample_lq(b, cfg, self.device, gen=self.gen)
        elif env_id in ("pyth_veh3dofconti", "pyth_veh3dofconti_errcstr"):
            # the errcstr data env inherits pyth_veh3dofconti's reset law (pyth_veh3dofconti_errcstr.py:19)
            self._draw = lambda b: ds.sample_veh3dofconti(b, P, self.device, gen=self.gen)
        elif env_id == "pyth_mobilerobot":
            self._draw = lambda b: ds.sample_mobilerobot(b, self.device, gen=self.gen)
        elif env_id == "veh3dof_tracking":
            self._draw = lambda b: ds.sample_veh3dof_tracking(b, P, self.device, gen=self.gen)
        elif env_id == "veh3dof_tracking_detour":
            self._draw = lambda b: ds.sample_veh3dof_tracking_detour(b, P, self.device, gen=self.gen)
        else:
            raise NotImplementedError(f"DeviceStateSampler: no on-device initial-state law for {env_id}")

    def sample(self, batch: int) -> Dict[str, torch.Tensor]:
        return self._draw(int(batch))


class DeviceEvaluator:
    """Batched closed-loop evaluation on the device (reference: gops/trainer/evaluator.py:45-86 runs
    `num_eval_episode` episodes one env.step at a time on the CPU and averages the returns).  Here all episodes run
    side by side through the fused single-step env model (`envmodel.forward`, one launch per step) with the
    evaluator's policy call `networks.policy(obs)` (deterministic mode of the action distribution; a
    FiniteHorizonPolicy is queried at virtual_t = 1, mlp.py:103-111).  An episode ends at `done` or after `max_step`
    steps (the data env's TimeLimit); rewards after `done` do not count."""

    def __init__(self, alg, sampler: DeviceStateSampler, num_eval_episode: int = 10, max_step: int = 200):
        self.alg, self.sampler = alg, sampler
        self.num_eval_episode, self.max_step = int(num_eval_episode), int(max_step)

    @torch.no_grad()
    def run_evaluation(self, iteration: int = 0) -> float:
        data = self.sampler.sample(self.num_eval_episode)
        obs, done = data["obs"], data["done"]
        info = {k: v for k, v in data.items() if k not in ("obs", "done")}
        ret = torch.zeros_like(done)
        alive = torch.ones_like(done)
        model = self.alg.envmodel
        for _ in range(self.max_step):
            act = self.alg.networks.policy(obs)
            obs, rew, d, info = model.forward(obs, act, done, info)
            ret += alive * rew
            done = d.to(ret.dtype)
            alive = alive * (1.0 - done)
            if float(alive.sum()) == 0.0:
                break
        return float(ret.mean())


class OnDeviceSerialTrainer:
    def __init__(self, alg, sampler: DeviceStateSampler, *, replay_batch_size: int, max_iteration: int,
                 log_save_interval: int = 100, apprfunc_save_interval: int = 0, save_folder: Optional[str] = None,
                 ini_network_dir: Optional[str] = None, sample_interval: int = 1,
                 evaluator: Optional["DeviceEvaluator"] = None, eval_interval: int = 0, **kwargs):
        self.alg, self.sampler, self.networks = alg, sampler, alg.networks
        if ini_network_dir is not None:
            self.networks.load_state_dict(torch.load(ini_network_dir))
        self.replay_batch_size, self.max_iteration = int(replay_batch_size), int(max_iteration)
        self.log_save_interval, self.apprfunc_save_interval = int(log_save_interval), int(apprfunc_save_interval)
        self.sample_interval = max(1, int(sample_interval))
        self.save_folder, self.iteration, self.history = save_folder, 0, []
        self.writer = None
        if save_folder is not None:
            os.makedirs(os.path.join(save_folder, "apprfunc"), exist_ok=True)
            try:
                from torch.utils.tensorboard import SummaryWriter
                self.writer = SummaryWriter(log_dir=save_folder, flush_secs=20)
            except Exception:
                self.writer = None
            with open(os.path.join(save_folder, "config.json"), "w") as f:
                json.dump({k: v for k, v in kwargs.items() if isinstance(v, (int, float, str, bool, list))}, f, indent=1)
        self._batch = None
        # evaluation + best-checkpoint bookkeeping of off_serial_trainer.py:113-141
        self.evaluator, self.eval_interval = evaluator, int(eval_interval)
        self.last_eval_iteration, self.best_tar = 0, -float("inf")
        self.start_time = time.time()

    def step(self):
        if self._batch is None or self.iteration % self.sample_interval == 0:
            self._batch = self.sampler.sample(self.replay_batch_size)
        self.networks.train()
        tb = self.alg.local_update(self._batch, self.iteration)
        self.networks.eval()
        if self.iteration % self.log_save_interval == 0:
            self.history.append((self.iteration, dict(tb)))
            if self.writer is not None:
                for tag, val in tb.items():
                    self.writer.add_scalar(tag, val, self.iteration)
        if self.apprfunc_save_interval and self.iteration % self.apprfunc_save_interval == 0:
            self.save_apprfunc()
        if self.evaluator is not None and self.eval_interval and \
                self.iteration - self.last_eval_iteration >= self.eval_interval:
            self.evaluate()
        self.iteration += 1
        return tb

    def evaluate(self) -> float:
        """Total average return of the current policy; keeps the best checkpoint as `apprfunc_{it}_opt.pkl` once a
        fifth of the iterations has passed (off_serial_trainer.py:126-141)."""
        self.last_eval_iteration = self.iteration
        total_avg_return = self.evaluator.run_evaluation(self.iteration)
        if self.writer is not None:
            self.writer.add_scalar(tb_tags["TAR of RL iteration"], total_avg_return, self.iteration)
        self.history.append((self.iteration, {tb_tags["TAR of RL iteration"]: total_avg_return}))
        if total_avg_return >= self.best_tar and self.iteration >= self.max_iteration / 5:
            self.best_tar = total_avg_return
            if self.save_folder is not None:
                folder = os.path.join(self.save_folder, "apprfunc")
                for fn in os.listdir(folder):
                    if fn.endswith("_opt.pkl"):
                        os.remove(os.path.join(folder, fn))
                sd = {k: v.detach().cpu() for k, v in self.networks.state_dict().items()}
                torch.save(sd, os.path.join(folder, f"apprfunc_{self.iteration}_opt.pkl"))
        return total_avg_return

    def train(self):
        while self.iteration < self.max_iteration:
            self.step()
        self.save_apprfunc()
        if self.writer is not None:
            self.writer.flush()

    def save_apprfunc(self):
        if self.save_folder is None:
            return
        sd = {k: v.detach().cpu() for k, v in self.networks.state_dict().items()}
        torch.save(sd, os.path.join(self.save_folder, "apprfunc", f"apprfunc_{self.iteration}.pkl"))
