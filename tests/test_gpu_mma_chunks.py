"""The fused mma.sync rollout kernel (csrc/kernel.cuh, rollout_kernel<M, HD, S, NT, ALG>) beyond the first sub-tile of a
CTA, against the fp64 oracle.

A launch runs min(#sub-tiles, SMs x occupancy) CTAs.  Each CTA takes a contiguous range of B / grid samples and works
through it in chunks of NT samples, each chunk in ceil(nv / S) sub-tiles of S samples.  The chunk configuration is
{S, NT} = {32, 128}, {64, 256} or {128, 512} for 64-wide nets (GOPS_B200_CFG = 2 / 1 / 0 forces one) and {32, 256} for
256-wide nets.  Every case here picks B from the grid of a warm-up launch so that, with n = B // grid samples per CTA:
  n >= 2 NT + 2 S   two full chunks, then a partial chunk of at least two sub-tiles;
  n mod S != 0      the last sub-tile of a CTA is ragged;
  B mod grid != 0   the ranges come in two lengths.
Then it asserts from the plans' launch records that this configuration and this shape actually ran (a forced
configuration that does not fit in shared memory silently falls back to the normal choice).

Bars are those of the single-sub-tile tests: loss 1e-4 relative, gradient 2e-4 relative L2 (1e-3 for the
pyth_veh3dofconti models), the interior-point variant's noise-floor rule, exact #done and safe counts."""
import numpy as np
import pytest
import torch

import test_gpu_constrained as cstr
import test_gpu_parity as base
import test_gpu_spil as spil
from oracle import gops_oracle as orc

pytestmark = pytest.mark.gpu

# GOPS_B200_CFG index of each 64-wide chunk configuration (kConfigs in csrc/gops_b200.cu)
CONFIGS = {(128, 512): "0", (64, 256): "1", (32, 128): "2"}
WIDE = (32, 256)                  # kWideConfig: 256-wide nets, not selectable
ALL = [(128, 512), (64, 256), (32, 128)]


def _sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _tag(cfg):
    return f"S{cfg[0]}xNT{cfg[1]}"


class Launches:
    """Every plan the algorithms of a test build (FusedADPMixin._plan), and the last launch of each."""

    def __init__(self, monkeypatch):
        from gops_b200.algorithm.base import FusedADPMixin
        self.monkeypatch, self.plans = monkeypatch, []
        plan_of = FusedADPMixin._plan

        def recording(alg, *a, **kw):
            plan = plan_of(alg, *a, **kw)
            if all(plan is not p for p in self.plans):
                self.plans.append(plan)
            return plan
        monkeypatch.setattr(FusedADPMixin, "_plan", recording)

    def force(self, cfg):
        if cfg in CONFIGS:
            self.monkeypatch.setenv("GOPS_B200_CFG", CONFIGS[cfg])

    def reset(self):
        self.plans.clear()

    def launched(self):
        """(grid, S, NT, smem bytes) of the last launch of every plan used since reset() that launched."""
        import ctypes as C
        from gops_b200 import _lib
        out = []
        for plan in self.plans:
            info = (C.c_int32 * 4)()
            _lib.check(_lib.lib().gops_b200_plan_launch_info(plan.handle, info))
            if info[0] > 0:
                assert plan.last_path() == "mma", plan.last_path()
                out.append((info[0], info[2], info[1], info[3]))
        assert out, "no fused rollout launch recorded"
        return out

    def batch(self, cfg, warmup):
        """Runs `warmup(B)` at a batch that fills every CTA slot and returns a batch B that gives the CTAs of every
        launch of that warm-up the shape of the module docstring."""
        S, NT = cfg
        self.reset()
        warmup(_sms() * 512)           # >= SMs x (2048 / NT) sub-tiles: more than CTA slots at any occupancy
        grids = set()
        for grid, s, nt, _ in self.launched():
            assert (s, nt) == cfg, ((s, nt), cfg)
            grids.add(grid)
        self.reset()

        def shaped(B, g):
            n = B // g
            return n >= 2 * NT + 2 * S and n % S != 0 and (n + 1) % S != 0 and B % g != 0
        g = max(grids)
        B = g * (2 * NT + 2 * S + S // 2) + g // 2
        while not all(shaped(B, g) for g in grids):
            B += 1
        return B

    def expect(self, label, B, cfg, shaped=True):
        """Asserts that every launch since reset() ran `cfg` (and, if `shaped`, with the CTA ranges of the docstring)."""
        S, NT = cfg
        for grid, s, nt, smem in self.launched():
            n = B // grid
            print(f"{label}: B={B} grid={grid} S={s} NT={nt} smem={smem} samples/CTA={n}"
                  f"{f'/{n + 1}' if B % grid else ''} chunks/CTA={-(-n // nt)}")
            assert (s, nt) == cfg, (label, (s, nt), cfg)
            if shaped:
                assert n >= 2 * NT + 2 * S and n % S != 0 and B % grid != 0, (label, B, grid)


@pytest.fixture
def launches(monkeypatch):
    """Algorithms ask for the mma.sync kernel; the launch records of their plans are kept."""
    from gops_b200.algorithm.base import FusedADPMixin
    monkeypatch.setattr(FusedADPMixin, "kernel_path", "mma")
    monkeypatch.delenv("GOPS_B200_CFG", raising=False)
    monkeypatch.delenv("GOPS_B200_ROLLOUT", raising=False)
    return Launches(monkeypatch)


# (env_id, algname, hidden activation (suffix 256: 256-wide nets), H, wrapper set of test_gpu_parity.WRAPPERS or None)
CASES = {
    "idp-FHADP-gelu": ("pyth_idpendulum", "FHADP", "gelu", 30, None),
    "idp-INFADP-elu": ("pyth_idpendulum", "INFADP", "elu", 8, None),
    "lq-INFADP-gelu": ("pyth_lq", "INFADP", "gelu", 8, None),
    "lq-FHADP-selu-s3a1clip": ("pyth_lq", "FHADP", "selu", 12, "s3a1-obs-rep2-clip"),
    "veh3dofconti-INFADP-relu": ("pyth_veh3dofconti", "INFADP", "relu", 6, None),
    "veh3dofconti-FHADP-gelu": ("pyth_veh3dofconti", "FHADP", "gelu", 10, None),
    "veh3dof_tracking-FHADP-elu": ("veh3dof_tracking", "FHADP", "elu", 10, None),
    "lq-INFADP-relu256": ("pyth_lq", "INFADP", "relu256", 5, None),
}
RUNS = ([("idp-FHADP-gelu", c) for c in ALL] + [("idp-INFADP-elu", c) for c in ALL]
        + [("lq-INFADP-gelu", c) for c in ALL] + [("lq-FHADP-selu-s3a1clip", (64, 256))]
        + [("veh3dofconti-INFADP-relu", c) for c in ALL[1:]] + [("veh3dofconti-FHADP-gelu", c) for c in ALL[1:]]
        + [("veh3dof_tracking-FHADP-elu", (64, 256)), ("lq-INFADP-relu256", WIDE)])


@pytest.mark.parametrize("case,cfg", [pytest.param(n, c, id=f"{n}-{_tag(c)}") for n, c in RUNS])
def test_against_oracle_fp64(launches, case, cfg):
    """Every sub-tile of a chunk, several chunks per CTA, ragged chunk tails: PEV and PIM (INFADP) or the FHADP policy
    gradient against the fp64 oracle, with done samples and the shaping wrappers."""
    env_id, algname, act, H, wrappers = CASES[case]
    wk = base.WRAPPERS[wrappers] if wrappers else base.SHAPING
    # the vehicle models' FHADP horizon is their observation's preview length; elsewhere a 1-step warm-up will do
    h_warm = H if (algname == "FHADP" and env_id != "pyth_idpendulum" and env_id != "pyth_lq") else 1
    launches.force(cfg)
    B = launches.batch(cfg, lambda b: base.check_against_oracle_fp64(env_id, algname, act, b, h_warm, wk))
    alg, n_done = base.check_against_oracle_fp64(env_id, algname, act, B, H, wk)
    launches.expect(case, B, cfg)
    if env_id == "pyth_idpendulum" and algname == "FHADP":
        got = float(alg.networks.policy.flat_params.gbuf[-2])      # tail = [loss | v-mean | #done | pad]
        print(f"{case}: #done {got:.0f} of {B} (oracle {n_done})")
        assert got == n_done, (got, n_done)


@pytest.mark.parametrize("algname,mode", [("FHADPExterior", "exterior"), ("FHADPLagrangian", "lagrangian"),
                                          ("FHADPInterior", "interior")])
def test_constrained_against_fp64_oracle(launches, algname, mode):
    """The interior variant's log barrier turns the fp32 round-off of a feasible sample next to the boundary into a
    gradient error without bound, and its bar is three times the fp32-vs-fp64 distance of the oracle on the same batch.
    Which draw puts a sample there is luck: at B = 88 770 (132 SMs) that distance is 0.34 for inputs drawn with seed B,
    1.3e-3 with seed 3.  Seed 3 keeps the bar meaningful."""
    cfg = (64, 256)
    launches.force(cfg)
    B = launches.batch(cfg, lambda b: cstr.check_against_fp64_oracle(algname, mode, b, seed=3))
    cstr.check_against_fp64_oracle(algname, mode, B, seed=3)
    launches.expect(algname, B, cfg)


def test_spil_against_fp64_oracle(launches):
    """Value pass (safe counts exact unless a constraint lies within 1e-4 of 0) and policy pass."""
    cfg = (64, 256)
    launches.force(cfg)
    B = launches.batch(cfg, spil.check_against_fp64_oracle)
    spil.check_against_fp64_oracle(B)
    launches.expect("SPIL", B, cfg)


def test_spil_update_at_its_benchmark_batch(launches):
    """B = 65536, the batch tools/bench_spil.py times, on the configuration the library picks: {128, 512} does not fit
    the 46-input nets in shared memory, so from SMs x 256 samples it is {64, 256}."""
    B = 65536
    spil.check_against_fp64_oracle(B)
    launches.expect("SPIL auto", B, (64, 256) if B >= _sms() * 256 else (32, 128), shaped=False)


def test_library_picks_the_largest_chunk_that_fills_every_sm(launches, monkeypatch):
    """pick_config without an override: {32, 128} below SMs x 256 samples, {64, 256} from there, {128, 512} from
    SMs x 512 (where it fits: idpendulum, not the 46-input vehicle nets); checked against the oracle at each side."""
    sms = _sms()
    for B, cfg in ((sms * 512 - 1, (64, 256)), (sms * 512, (128, 512))):
        launches.reset()
        base.check_against_oracle_fp64("pyth_idpendulum", "FHADP", "gelu", B, 4, base.SHAPING)
        launches.expect("idp mma", B, cfg, shaped=False)
    from gops_b200.algorithm.base import FusedADPMixin
    monkeypatch.setattr(FusedADPMixin, "kernel_path", "auto")     # the vehicle models have no wgmma kernel
    for B, cfg in ((sms * 256 - 1, (32, 128)), (sms * 256, (64, 256))):
        launches.reset()
        base.check_against_oracle_fp64("pyth_veh3dofconti", "FHADP", "gelu", B, 10, base.SHAPING)
        launches.expect("veh3dofconti auto", B, cfg, shaped=False)


def _idp_fhadp(H, **wrappers):
    from gops_b200.create_pkg.create_alg import create_alg
    kw, _ = base.make_kwargs("fhadp_idp_h30")
    kw.update(pre_horizon=H, **wrappers)
    torch.manual_seed(H)
    return create_alg(**kw)


def _idp_inputs(B, seed, dev):
    data = orc.sample_inputs("pyth_idpendulum", B, seed=seed)
    data["done"][::7] = 1.0
    return {k: v.to(dev) for k, v in data.items()}


@pytest.mark.parametrize("cfg", [(128, 512), (64, 256)], ids=_tag)
def test_trace_against_oracle(launches, cfg):
    """The per-step trace (observation, action, reward, done) of every sample against the oracle's rollout."""
    import ctypes as C
    from gops_b200 import _lib
    from gops_b200.env.fused import make_batch
    H = 12
    alg = _idp_fhadp(H, **base.SHAPING)
    dev, pol = alg._device(), alg.networks.policy

    def trace(data):
        B = data["obs"].shape[0]
        plan = alg._plan(_lib.ALG_FHADP, pol, None, H, alg.gamma)
        o, a = torch.empty(H, B, 6, device=dev), torch.empty(H, B, 1, device=dev)
        r, d = torch.empty(H, B, device=dev), torch.empty(H, B, device=dev)
        keep = []
        b = make_batch(alg.envmodel.unwrapped, data["obs"], data["done"], {}, keep)
        _lib.check(_lib.lib().gops_b200_rollout_trace(plan.handle, C.byref(b), _lib.ptr(pol.flat_params.sync()),
                                                     _lib.ptr(o), _lib.ptr(a), _lib.ptr(r), _lib.ptr(d),
                                                     _lib.stream_ptr()))
        torch.cuda.synchronize()
        return o.cpu().numpy(), a.cpu().numpy(), r.cpu().numpy(), d.cpu().numpy()

    launches.force(cfg)
    B = launches.batch(cfg, lambda b: trace(_idp_inputs(b, 1, dev)))
    data = _idp_inputs(B, 3, dev)
    o, a, r, d = trace(data)
    launches.expect("trace", B, cfg)
    spec = base._oracle_nets(alg, "gelu", torch.float64)(pol, "pi", True)
    env = orc.create_env_model("pyth_idpendulum", dtype=torch.float64, **base.SHAPING)
    ref = []
    with torch.no_grad():
        orc.fhadp_loss(spec, env, {k: v.cpu().double() for k, v in data.items()}, H, alg.gamma, trace=ref)
    for k, (o_k, a_k, r_k, d_k) in enumerate(ref):
        assert (d[k] == d_k.double().numpy()).all(), f"step {k}: termination differs from the oracle"
        np.testing.assert_allclose(a[k], a_k.numpy(), rtol=1e-4, atol=2e-6, err_msg=f"step {k}")
        np.testing.assert_allclose(o[k], o_k.numpy(), rtol=2e-4, atol=2e-4, err_msg=f"step {k}")
        np.testing.assert_allclose(r[k], r_k.numpy(), rtol=2e-4, atol=2e-3, err_msg=f"step {k}")


@pytest.mark.parametrize("cfg", ALL, ids=_tag)
def test_deterministic_and_all_done(launches, cfg):
    """The same call twice gives the same gradient bit for bit; a batch that arrives done gives exactly zero."""
    alg = _idp_fhadp(8, reward_scale=1.0)
    dev = alg._device()

    def grad(data):
        alg._compute_gradient(data)
        torch.cuda.synchronize()
        return alg.networks.policy.flat_params.gbuf.clone()

    launches.force(cfg)
    B = launches.batch(cfg, lambda b: grad(_idp_inputs(b, 1, dev)))
    data = _idp_inputs(B, 5, dev)
    g1, g2 = grad(data), grad(data)
    launches.expect("determinism", B, cfg)
    n = g1.numel() - 4
    assert float(g1[:n].abs().max()) > 0.0
    assert torch.equal(g1, g2), "the fused update must be bit-deterministic"
    g0 = grad(dict(data, done=torch.ones_like(data["done"])))
    assert float(g0[:n].abs().max()) == 0.0
    assert float(g0[n]) == 0.0 and float(g0[n + 2]) == B      # reward_scale 1, shift 0: masked samples pay nothing
