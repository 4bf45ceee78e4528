#!/usr/bin/env python
"""Regenerate tests/golden/amis_resident/*.npz: inputs and outputs of the fused LM + AMIS call on short point sets (the
resident AMIS kernel) under the single-CTA SIMT emulator, built from the kernel sources of a given tree.

    python tools/make_amis_resident_golden.py --tree <source tree> [--out tests/golden/amis_resident]

The fixture pins the resident kernel's results bit for bit (tests/test_amis_resident_golden_simt_cpu.py), so regenerate it
from the commit whose results it should hold, e.g. a `git worktree` of that commit.  The emulator shim and the Python
layers come from this repository; only the kernel sources (csrc/, include/) come from --tree."""
import argparse
import contextlib
import ctypes
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "epro-pnp_b200"))

from epropnp_b200 import capi, native  # noqa: E402
from epropnp_b200.synth import make_noise, make_problem  # noqa: E402

# (samples per iteration S, iterations I, points N, injected noise): S covers one sample per CTA, S < 64, S = 64, S not a
# multiple of 64 or 128, S = 128 and S > 128; N covers odd N and N < 8.
CASES = [(1, 4, 37, False), (40, 4, 5, True), (64, 2, 64, False), (100, 3, 37, True), (128, 2, 24, False),
         (200, 2, 7, False), (128, 2, 37, True)]
B = 2


def build_emulated(tree, out_dir):
    shim = os.path.join(REPO, "tests", "simt_emul")
    out = os.path.join(out_dir, "libepropnp_simt.so")
    cmd = ["g++", "-std=c++20", "-O2", "-mfma", "-ffp-contract=fast", "-x", "c++", "-DEPNP_SIMT_EMUL", "-fPIC", "-shared",
           "-I", shim, "-I", os.path.join(tree, "include"), "-I", os.path.join(tree, "epro-pnp_b200", "csrc"), "-o", out,
           os.path.join(tree, "epro-pnp_b200", "csrc", "pnp_kernels.cu")]
    subprocess.run(cmd, check=True)
    h = ctypes.CDLL(out)
    for name, (res, args) in capi._SIGNATURES.items():
        fn = getattr(h, name)
        fn.restype, fn.argtypes = res, args
    return h


def use_emulator(h):
    """Point the ctypes layer at the emulated library (as tests/simt_native.install does for one test)."""
    capi._lib = h
    native._need_cuda = lambda t, what: None
    native.stream_ptr = lambda device=None: None
    torch.cuda.device = lambda device=None: contextlib.nullcontext()
    torch.cuda.synchronize = lambda device=None: None


def case_inputs(dof, bounded, S, I, N, injected, k):
    pc = make_problem(B, N, seed=100 + k, dof=dof)
    d = {name: pc[name].contiguous() for name in ("x3d", "x2d", "w2d", "cam_mats", "pose_init")}
    if bounded:
        d["lb"] = (pc["x2d"].amin(1) + 2.0).contiguous()
        d["ub"] = (pc["x2d"].amax(1) - 2.0).contiguous()
    if injected:
        n3, chi2, rot = make_noise(B, S * I, seed=200 + k, dof=dof)
        d["noise_n3"], d["noise_chi2"], d["noise_rot"] = n3.contiguous(), chi2.contiguous(), rot.contiguous()
    return d


def run_case(d, dof, S, I):
    """The fused LM + AMIS call on the inputs `d` (a dict of CPU tensors) -> dict of output tensors."""
    delta = native.adaptive_delta(d["x2d"], d["w2d"], 0.5)
    prob = native.Problem(d["x3d"], d["x2d"], d["w2d"], d["cam_mats"], d.get("lb"), d.get("ub"), delta)
    p = native.default_params(dof, lm_iter=3, mc_samples=S * I, mc_iter=I)
    noise = (d["noise_n3"], d["noise_chi2"], d["noise_rot"]) if "noise_n3" in d else None
    out = native.lm_amis_fused(prob, d["pose_init"], p, noise=noise, seed=11, want_proposals=True)
    return {k: out[k] for k in ("pose_opt", "pose_samples", "logw", "proposals")}


def case_name(S, I, N, injected):
    return f"S{S}_I{I}_N{N}_{'injected' if injected else 'philox'}"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--tree", required=True, help="source tree whose kernels produce the fixture")
    ap.add_argument("--out", default=os.path.join(REPO, "tests", "golden", "amis_resident"))
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        use_emulator(build_emulated(os.path.abspath(a.tree), tmp))
        os.makedirs(a.out, exist_ok=True)
        for dof in (6, 4):
            for bounded in (False, True):
                arrays = {}
                for k, (S, I, N, injected) in enumerate(CASES):
                    d = case_inputs(dof, bounded, S, I, N, injected, k)
                    res = run_case(d, dof, S, I)
                    name = case_name(S, I, N, injected)
                    arrays.update({f"{name}/in/{key}": v.numpy() for key, v in d.items()})
                    arrays.update({f"{name}/out/{key}": v.numpy() for key, v in res.items()})
                path = os.path.join(a.out, f"dof{dof}_{'bounded' if bounded else 'unbounded'}.npz")
                np.savez_compressed(path, **arrays)
                print("wrote", path)


if __name__ == "__main__":
    main()
