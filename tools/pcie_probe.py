#!/usr/bin/env python
"""Host <-> device copy ceiling of the box the bench runs on (pinned memory, CUDA events):
H2D alone, D2H alone, and both directions at once, at the chunk sizes of the end-to-end path.

bench.py's `e2e` number moves 59 MB in and 68 MB out per 4096-object step; whether its rate is the link's limit or
the pipeline's is what this tool answers (`python tools/pcie_probe.py > pcie_probe.json`)."""
import json
import sys

import torch


def rate(fn, nbytes, iters=20):
    torch.cuda.synchronize()
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return nbytes * iters / (a.elapsed_time(b) * 1e-3) / 1e9


def main():
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    dev = torch.device("cuda:0")
    out = {"device": torch.cuda.get_device_name(0), "sizes_MB": {}}
    s_in, s_out = torch.cuda.Stream(), torch.cuda.Stream()
    for mb in (4, 16, 64, 256):
        n = mb << 20
        h_in = torch.empty(n, dtype=torch.uint8).pin_memory()
        h_out = torch.empty(n, dtype=torch.uint8).pin_memory()
        d_in = torch.empty(n, dtype=torch.uint8, device=dev)
        d_out = torch.empty(n, dtype=torch.uint8, device=dev)

        def h2d():
            d_in.copy_(h_in, non_blocking=True)

        def d2h():
            h_out.copy_(d_out, non_blocking=True)

        def both():
            cur = torch.cuda.current_stream()
            s_in.wait_stream(cur)
            s_out.wait_stream(cur)
            with torch.cuda.stream(s_in):
                d_in.copy_(h_in, non_blocking=True)
            with torch.cuda.stream(s_out):
                h_out.copy_(d_out, non_blocking=True)
            cur.wait_stream(s_in)
            cur.wait_stream(s_out)

        out["sizes_MB"][mb] = {"h2d_GBps": round(rate(h2d, n), 2), "d2h_GBps": round(rate(d2h, n), 2),
                               "duplex_each_GBps": round(rate(both, n), 2)}
    # the same copies with the host buffers first-touched on the GPU's NUMA node (bench.py EPNP_E2E_NUMA=1)
    import os
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from bench import gpu_local_cpus
    n = 64 << 20
    with gpu_local_cpus(0, True) as numa:
        h_in = torch.empty(n, dtype=torch.uint8).pin_memory()
        h_out = torch.empty(n, dtype=torch.uint8).pin_memory()
    d = torch.empty(n, dtype=torch.uint8, device=dev)
    out["gpu_numa_local_64MB"] = {"cpus_bound": numa.applied, "cpus_total": os.cpu_count(),
                                  "h2d_GBps": round(rate(lambda: d.copy_(h_in, non_blocking=True), n), 2),
                                  "d2h_GBps": round(rate(lambda: h_out.copy_(d, non_blocking=True), n), 2)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
