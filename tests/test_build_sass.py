"""The built objects must contain the instructions the design claims (checked on the SASS of the sm_90a cubins, no GPU
needed): warpgroup tensor-core MMAs (wgmma) in the tensor-core rollout, layer-wise and inference kernels, TF32 mma.sync
in the fused mma.sync rollout kernel, TMA bulk copies for the weight staging."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _count(obj, needles):
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    counts = dict.fromkeys(needles, 0)
    p = subprocess.Popen([exe, "-sass", obj], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
    for line in p.stdout:
        for n in needles:
            if n in line:
                counts[n] += 1
    p.wait()
    return counts


def _objects():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as g
    g.build()
    return os.path.join(ROOT, "build", "obj")


def test_rollout_objects_carry_tcgen05_tma_and_tf32_mma():
    """(Name kept from the Blackwell build: the tensor-core rollout kernel is now wgmma.)"""
    c = _count(os.path.join(_objects(), "kernels_idp.o"), ["HGMMA", "WARPGROUP.DEPBAR", "HMMA.1688.F32.TF32", "UBLKCP", "SYNCS"])
    assert c["HGMMA"] > 100, c            # wgmma (rollout_tc2: BF16x3 layer / delta / weight-gradient products)
    assert c["WARPGROUP.DEPBAR"] > 8, c   # wgmma.wait_group
    assert c["HMMA.1688.F32.TF32"] > 100, c      # mma.sync 3xTF32 path
    assert c["UBLKCP"] > 4, c             # cp.async.bulk weight staging
    assert c["SYNCS"] > 8, c              # mbarrier transaction counts / phase checks of the staging


def test_layerwise_objects_carry_tcgen05():
    """dense_tc.o: the forward / dgrad / wgrad GEMMs of the layer-wise path (wgmma; name kept from the Blackwell build);
    kernels_vehtrack.o only hosts the per-step kernels of C3 (its dense products run in dense_tc.o)."""
    c = _count(os.path.join(_objects(), "dense_tc.o"), ["HGMMA", "WARPGROUP.DEPBAR", "UBLKCP"])
    assert c["HGMMA"] >= 90 and c["WARPGROUP.DEPBAR"] >= 5 and c["UBLKCP"] >= 4, c


def test_inference_object_carries_tcgen05():
    """The 64-wide inference kernel (wgmma TF32; name kept from the Blackwell build)."""
    c = _count(os.path.join(_objects(), "gops_b200.o"), ["HGMMA.64x64x8.F32.TF32", "WARPGROUP.DEPBAR", "UBLKCP"])
    assert c["HGMMA.64x64x8.F32.TF32"] >= 18 and c["WARPGROUP.DEPBAR"] >= 2 and c["UBLKCP"] >= 2, c
