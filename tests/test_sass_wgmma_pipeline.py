"""The wgmma convolution kernels keep their wgmma pipeline in the compiled code (no GPU needed).

When ptxas cannot keep several wgmma of a warpgroup in flight (for instance because an accumulator register would sit
at different positions in the register tuples of two wgmma), it reports C7511 and follows EVERY wgmma with a full wait
(`WARPGROUP.DEPBAR.LE gsb0, 0x0`), so that each small MMA pays its whole latency.  The kernels themselves only wait for
all of their wgmma once per tile (and otherwise with `wgmma.wait_group 1`), so a pipelined build has many HGMMA per
full wait.  This reads the SASS of the built library and fails if a convolution kernel lost its pipeline."""
import importlib.util
import os
import re
import subprocess
from collections import defaultdict

from conftest import PKG

MIN_HGMMA_PER_FULL_WAIT = 6
FULL_WAIT = re.compile(r'WARPGROUP\.DEPBAR\.LE\s+gsb0\s*,\s*0x0\b')


def _built_library():
    spec = importlib.util.spec_from_file_location('vr_b200_build', os.path.join(PKG, 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build(), os.path.join(os.path.dirname(mod.NVCC), 'cuobjdump')


def _wgmma_counts(lib, cuobjdump):
    """{mangled kernel name: [HGMMA count, full-wait count]} of every function in lib that issues wgmma"""
    sass = subprocess.run([cuobjdump, '-sass', lib], capture_output=True, text=True, check=True).stdout
    counts = defaultdict(lambda: [0, 0])
    fn = None
    for line in sass.splitlines():
        m = re.match(r'\s*Function\s*:\s*(\S+)', line)
        if m:
            fn = m.group(1)
        elif fn is not None and 'HGMMA' in line:
            counts[fn][0] += 1
        elif fn is not None and FULL_WAIT.search(line):
            counts[fn][1] += 1
    return {k: v for k, v in counts.items() if v[0]}


def test_conv_kernels_keep_the_wgmma_pipeline():
    lib, cuobjdump = _built_library()
    counts = _wgmma_counts(lib, cuobjdump)
    rows = {k: v for k, v in counts.items() if 'conv_tc_rows_kernel' in k}
    generic = {k: v for k, v in counts.items() if 'conv_tc_kernel' in k}
    assert len(rows) == 6, sorted(rows)   # BN = 16 / 32 / 64, with and without the fused upsample
    assert generic, sorted(counts)
    serialised = {k: v for k, v in sorted({**rows, **generic}.items())
                  if v[0] < MIN_HGMMA_PER_FULL_WAIT * max(v[1], 1)}
    assert not serialised, 'wgmma serialised (kernel: [HGMMA, full waits]): %s' % serialised
