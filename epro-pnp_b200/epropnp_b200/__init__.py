"""epropnp_b200 -- native side of the H100 EPro-PnP layer: build helper, ctypes binding of
libepropnp_b200.so (include/epropnp_b200.h), synthetic inputs and the batch-sharding helper.
The drop-in Python surface of the reference lives next to this package in `epropnp/`."""
from .capi import EpnpParams, default_params, lib, lib_path, NativeError  # noqa: F401
