"""TEST-ONLY: simt_native for the cluster-split kernels.  Builds epro-pnp_b200/csrc/pnp_kernels.cu with
`g++ -DEPNP_SIMT_EMUL` against the cluster emulator in tests/simt_cluster/ (the single-CTA emulator of tests/simt_emul
extended to thread-block clusters; its math_constants.h is shared) and points the ctypes layer at it for one test.
Under the single-CTA emulator the split entry points report EPNP_ERR_UNSUPPORTED."""
import ctypes
import hashlib
import os
import subprocess

import simt_native
from epropnp_b200 import build, capi

_HERE = os.path.dirname(os.path.abspath(__file__))
_SHIM = os.path.join(_HERE, "simt_cluster")
_handles = {}


def build_emulated(flags=()):
    flags = tuple(flags)
    tag = hashlib.sha1(" ".join(flags).encode()).hexdigest()[:8] if flags else "default"
    out = os.path.join(build.LIB_DIR, f"libepropnp_simt_cluster_{tag}.so")
    src = os.path.join(build.CSRC, "pnp_kernels.cu")
    deps = build.kernel_sources() + [os.path.join(_SHIM, "cuda_runtime.h"), os.path.join(simt_native._SHIM, "math_constants.h")]
    os.makedirs(build.LIB_DIR, exist_ok=True)
    if build._newer(out, deps):
        # -fno-gnu-unique: the emulator's function-local statics (simt::state() ...) must stay private to this library;
        # as GNU-unique symbols they would bind process-wide to the single-CTA emulator's, whose layout differs
        cmd = ["g++", "-std=c++20", "-O2", "-mfma", "-ffp-contract=fast", "-fno-gnu-unique", "-x", "c++", "-DEPNP_SIMT_EMUL",
               *flags, "-fPIC", "-shared", "-I", _SHIM, "-I", simt_native._SHIM, "-I", build.INCLUDE, "-I", build.CSRC, "-o", out, src]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("g++ (SIMT cluster emulation build) failed:\n" + r.stdout + r.stderr)
    return out


def handle(flags=()):
    flags = tuple(flags)
    if flags not in _handles:
        h = ctypes.CDLL(build_emulated(flags))
        for name, (res, args) in capi._SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype, fn.argtypes = res, args
        _handles[flags] = h
    return _handles[flags]


def install(monkeypatch, flags=()):
    """simt_native.install with the cluster emulator's library in place of the single-CTA one."""
    dev = simt_native.install(monkeypatch)
    monkeypatch.setattr(capi, "_lib", handle(flags))
    return dev
