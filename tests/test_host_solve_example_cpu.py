"""examples/host_solve_c.c, a C99 host of epnp_solve_host_f32, builds with gcc against include/epropnp_b200.h, links to
the library and passes its device-free checks: EpnpInit's layout, the workspace query and the argument refusals."""
import os
import subprocess

from epropnp_b200 import build, capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_host_solve_example_links_and_runs(tmp_path):
    build.build_library()
    exe = str(tmp_path / "host_solve_c")
    lib_dir = os.path.dirname(capi.lib_path())
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "examples", "host_solve_c.c"), "-o", exe, "-L", lib_dir, "-lepropnp_b200",
                    "-Wl,-rpath," + lib_dir], check=True)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr


def test_ctypes_layout_matches_the_header():
    assert capi.EpnpInit.seed.offset == 16 and capi.EpnpInit.rslm.offset == 32
    assert capi.EpnpInit.conf_quantile.offset == 24
