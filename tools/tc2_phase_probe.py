"""Cycles per phase of the fused wgmma rollout kernel on the headline update (FHADP idpendulum, GELU 64x64, H = 30,
batch 2^18), from a library built with the phase probe of gops_b200/csrc/tc2_probe.cuh.

    python tools/tc2_phase_probe.py build OUT.so [--csrc DIR]   # a probe build of the sources in DIR (default: this tree)
    python tools/tc2_phase_probe.py run OUT.so [--iters N] [--json FILE]

`build` compiles every translation unit with -DGOPS_TC2_PHASE_PROBE into OUT.so (objects in a temporary directory);
the library under gops_b200/lib is not touched.  `--csrc` takes the csrc directory of another checkout, so that two
versions of the kernel can be probed side by side.  `run` loads OUT.so in a child process, runs `--warmup` + `--iters`
updates and prints the mean clock64() cycles per warpgroup and horizon step of each phase (thread 0 of each warpgroup
stamps; the phases are listed in tc2_probe.cuh).  The stamps add a few instructions and registers to the kernel, so the
probe's totals run somewhat above the unprobed kernel's; compare probe builds with each other.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["fwd_l1", "fwd_l2", "fwd_dyn", "rev_l1", "rev_adj", "rev_l2", "rev_d2", "rev_d1"]
LINE = re.compile(r"tc2probe alg=(\d+) wgs=(\d+) fwd_steps=(\d+) rev_steps=(\d+) (.*)")


def build(out, csrc):
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = [f for f in ge.NVCC_FLAGS if not f.startswith("-I")]
    flags += ["-I" + os.path.join(os.path.dirname(os.path.dirname(csrc)), "include"), "-I" + csrc,
              "-DGOPS_TC2_PHASE_PROBE"]
    sources = sorted(f for f in os.listdir(csrc) if f.endswith(".cu"))
    with tempfile.TemporaryDirectory() as tmp:
        objs = [os.path.join(tmp, s[:-3] + ".o") for s in sources]

        def run(cmd):
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)

        with ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1))) as ex:
            list(ex.map(run, [[nvcc] + flags + ["-c", os.path.join(csrc, s), "-o", o] for s, o in zip(sources, objs)]))
        run([nvcc, "-shared", "-o", os.path.abspath(out)] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    print(f"probe library: {out}")


def child(B, H, warmup, iters):
    """one process: the probe lines are printed by the kernel on the C stdout"""
    import numpy as np
    import torch
    sys.path.insert(0, ROOT)
    from gops_b200.create_pkg.create_alg import create_alg
    from gops_b200.trainer import device_sampler as ds
    kw = dict(env_id="pyth_idpendulum", algorithm="FHADP", seed=0, trainer="off_serial_trainer", use_gpu=True,
              action_type="continu", obsv_dim=6, action_dim=1, action_high_limit=np.ones(1, np.float32),
              action_low_limit=-np.ones(1, np.float32), policy_func_name="FiniteHorizonPolicy",
              policy_func_type="MLP", policy_hidden_sizes=[64, 64], policy_hidden_activation="gelu",
              policy_act_distribution="default", policy_learning_rate=1e-4, value_func_type="MLP", pre_horizon=H)
    torch.manual_seed(0)
    alg = create_alg(**kw)
    alg.kernel_path = "tc"
    data = ds.sample_idpendulum(B, "cuda", 1)
    for _ in range(warmup + iters):
        alg._compute_gradient(data)
        torch.cuda.synchronize()
    assert alg.last_kernel_path() == "tc", alg.last_kernel_path()


def run(lib, B, H, warmup, iters, json_out):
    env = dict(os.environ, GOPS_B200_LIB=os.path.abspath(lib))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "_child", str(B), str(H), str(warmup), str(iters)],
                       env=env, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("probe run failed:\n" + r.stdout[-4000:] + r.stderr[-4000:])
    rows = []
    for ln in r.stdout.splitlines():
        m = LINE.search(ln)
        if m and int(m.group(1)) == 0:
            kv = dict(x.split("=") for x in m.group(5).split())
            rows.append((int(m.group(3)), int(m.group(4)), {k: int(v) for k, v in kv.items()}))
    if len(rows) != warmup + iters:
        raise RuntimeError(f"expected {warmup + iters} probe lines of the FHADP kernel, got {len(rows)}:\n{r.stdout[-4000:]}")
    rows = rows[warmup:]
    fs, rs = sum(x[0] for x in rows), sum(x[1] for x in rows)
    res = {ph: sum(x[2][ph] for x in rows) / (fs if ph.startswith("fwd") else rs) for ph in PHASES}
    res["fwd_total"] = sum(v for k, v in res.items() if k.startswith("fwd"))
    res["rev_total"] = sum(res[k] for k in PHASES if k.startswith("rev"))
    print(f"{lib}: mean cycles per warpgroup-step (batch {B}, H {H}, {iters} updates)")
    for k, v in res.items():
        print(f"  {k:10s} {v:10.0f}")
    if json_out:
        with open(json_out, "w") as f:
            json.dump(dict(lib=lib, batch=B, horizon=H, iters=iters, cycles_per_step=res), f, indent=1)


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "_child":
        child(*(int(a) for a in sys.argv[2:6]))
        return
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("mode", choices=["build", "run"])
    ap.add_argument("lib")
    ap.add_argument("--csrc", default=os.path.join(ROOT, "gops_b200", "csrc"))
    ap.add_argument("--batch", type=int, default=1 << 18)
    ap.add_argument("--horizon", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if a.mode == "build":
        build(a.lib, os.path.abspath(a.csrc))
    else:
        run(a.lib, a.batch, a.horizon, a.warmup, a.iters, a.json)


if __name__ == "__main__":
    main()
