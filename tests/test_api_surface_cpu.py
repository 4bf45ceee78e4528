"""Drop-in check by introspection: every public function, class, method and static method of the six reference modules
on the path (epropnp.epropnp, .levenberg_marquardt, .camera, .cost_fun, .common, .distributions) exists under the same
name in the package, and every parameter of the reference signature is present in ours, in the same order, with the
same default (ours may append optional keyword arguments).  The reference's surface is stored in
tests/golden/api_surface/reference.json.gz, dumped from the unmodified reference with the pyro shim:

    python tests/test_api_surface_cpu.py <reference checkout>      # rewrites the stored surface
"""
import gzip
import json
import os
import subprocess
import sys

from conftest import ROOT

MODULES = ("epropnp.epropnp", "epropnp.levenberg_marquardt", "epropnp.camera", "epropnp.cost_fun", "epropnp.common",
           "epropnp.distributions")
GOLDEN = os.path.join(ROOT, "tests", "golden", "api_surface", "reference.json.gz")

_DUMP = r'''
import importlib, inspect, json, sys
def params(f):
    try:
        return [[p.name, p.kind.name, None if p.default is inspect.Parameter.empty else repr(p.default)]
                for p in inspect.signature(f).parameters.values()]
    except (TypeError, ValueError):
        return None
out = {}
for m in sys.argv[2:]:
    mod = importlib.import_module(m)
    for n, o in vars(mod).items():
        if n.startswith('_'):
            continue
        own = getattr(o, '__module__', None) == m
        if inspect.isclass(o) and (own or sys.argv[1] == 'all'):
            for kls in (o.__mro__ if sys.argv[1] == 'all' else (o,)):
                for mn, mo in vars(kls).items():
                    if mn.startswith('__') and mn != '__init__':
                        continue
                    f = mo.__func__ if isinstance(mo, (staticmethod, classmethod)) else mo
                    if callable(f):
                        out.setdefault(f'{m}:{n}.{mn}', params(f))
        elif callable(o) and not inspect.isclass(o) and (own or sys.argv[1] == 'all'):
            out[f'{m}:{n}'] = params(o)
print(json.dumps(out))
'''


def _surface(paths, mode):
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(paths))
    r = subprocess.run([sys.executable, "-c", _DUMP, mode, *MODULES], capture_output=True, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_every_public_name_and_parameter_of_the_reference_exists_here():
    with gzip.open(GOLDEN, "rt") as f:
        ref = json.load(f)
    ours = _surface([os.path.join(ROOT, "epro-pnp_b200"), ROOT], "all")
    assert len(ref) > 60
    missing = sorted(k for k in ref if k not in ours)
    assert not missing, missing
    problems = []
    for name, want in ref.items():
        have = ours[name]
        if want is None or have is None:
            continue
        if any(kind in ("VAR_POSITIONAL", "VAR_KEYWORD") for _, kind, _ in want) and len(want) <= 3 and want[-1][0] in ("args", "kwargs"):
            continue                                           # the base class's abstract (*args, **kwargs) stubs
        fixed = [p for p in want if p[1] not in ("VAR_POSITIONAL", "VAR_KEYWORD")]
        ours_fixed = [p for p in have if p[1] not in ("VAR_POSITIONAL", "VAR_KEYWORD")]
        if ours_fixed[:len(fixed)] != fixed:
            problems.append((name, fixed, ours_fixed))
        elif any(extra[2] is None for extra in ours_fixed[len(fixed):]):
            problems.append((name, "extra parameter without a default", ours_fixed[len(fixed):]))
    assert not problems, problems


if __name__ == "__main__":
    surface = _surface([os.path.join(ROOT, "oracle", "pyro_shim"), os.path.abspath(sys.argv[1])], "own")
    os.makedirs(os.path.dirname(GOLDEN), exist_ok=True)
    with gzip.GzipFile(GOLDEN, "wb", mtime=0) as f:
        f.write(json.dumps(surface, sort_keys=True, separators=(",", ":")).encode())
