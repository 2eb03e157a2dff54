#!/usr/bin/env python
"""The ctc_rec_kernel<K, BACK> instantiations that one CTC forward + backward launches at each recursion width
(target lengths 1, 128, 256, 512, 1024, 2048: K = 1 .. 32), read with torch.profiler; exits 1 unless all 12 appear.
usage: python tools/ctc_kernel_names.py"""
import re
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from tests.ctc_util import repeats  # noqa: E402
from tests.test_gpu_ctc_widths import _call, _pack, _target  # noqa: E402
from b200asr import _lib as L  # noqa: E402

lib = L.load(check_device=True)
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for lmax in (1, 128, 256, 512, 1024, 2048):
        y = _target(np.random.default_rng(lmax), lmax, 5)
        T = lmax + repeats(y) + 2
        _call(lib, torch.randn(1, T, 5), _pack([y], 5), [T], [lmax])
names = {e.name() for e in prof.profiler.kineto_results.events() if e.device_type() == torch.autograd.DeviceType.CUDA}
seen = sorted({m.groups() for n in names for m in [re.search(r"ctc_rec_kernel<(\d+), (true|false)>", n)] if m},
              key=lambda g: (int(g[0]), g[1]))
for k, back in seen:
    print(f"ctc_rec_kernel<{k}, {back}>")
want = {(str(k), b) for k in (1, 2, 4, 8, 16, 32) for b in ("true", "false")}
print(f"{len(seen)} of 12 instantiations launched")
sys.exit(0 if set(seen) == want else 1)
