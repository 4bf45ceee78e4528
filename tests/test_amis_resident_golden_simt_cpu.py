"""The resident AMIS kernel (short point sets, one CTA per object) under the single-CTA SIMT emulator, held bit for bit
to committed outputs (tests/golden/amis_resident, written by tools/make_amis_resident_golden.py).  A change to the
kernel that is meant to keep its results, such as a new thread mapping or a re-tuned sweep, has to keep these bits.
The cases cover S = M / I = 1, below 64, at 64, not a multiple of 64 or 128, at 128 and above 128, odd N and N < 8,
bounded and unbounded cameras, Philox and injected noise, 6DoF and 4DoF."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

import simt_native

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import make_amis_resident_golden as golden  # noqa: E402

FIXTURES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "amis_resident", "*.npz")))


def _cases(path):
    z = np.load(path)
    for name in sorted({k.split("/")[0] for k in z.files}):
        d = {k.split("/", 2)[2]: torch.from_numpy(z[k]) for k in z.files if k.startswith(name + "/in/")}
        want = {k.split("/", 2)[2]: z[k] for k in z.files if k.startswith(name + "/out/")}
        S, I = int(name.split("_")[0][1:]), int(name.split("_")[1][1:])
        yield name, d, S, I, want


def test_fixture_is_complete():
    assert [os.path.basename(p) for p in FIXTURES] == [
        "dof4_bounded.npz", "dof4_unbounded.npz", "dof6_bounded.npz", "dof6_unbounded.npz"]


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p)[:-4] for p in FIXTURES])
def test_resident_kernel_matches_the_fixture_bit_for_bit(monkeypatch, path):
    simt_native.install(monkeypatch)
    dof = 6 if os.path.basename(path).startswith("dof6") else 4
    n = 0
    for name, d, S, I, want in _cases(path):
        got = golden.run_case(d, dof, S, I)
        for k, w in want.items():
            g = got[k].numpy()
            assert g.shape == w.shape, (name, k)
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), (name, k)
        n += 1
    assert n == len(golden.CASES)
