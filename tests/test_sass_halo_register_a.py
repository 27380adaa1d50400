"""The halo-tile convolution reads A from registers, keeps its wgmma pipeline and has no local memory (no GPU needed).

conv_tc_halo_kernel loads one halo tile per channel chunk and gathers the A fragments of every tap from it with
ldmatrix, so every HGMMA must take A from registers (`HGMMA ... R, R, gdesc`).  Each (tap, k-step) is one commit group
and the kernel only waits for all of its wgmma once per tile, so a pipelined build has many HGMMA per full
`WARPGROUP.DEPBAR.LE gsb0, 0x0`; ptxas falls back to one full wait per HGMMA when the accumulators and fragments do not
fit (C7512).  Spilled accumulators or fragments would show up as STL / LDL: at MB = 2 the consumers need the registers
setmaxnreg gives them, and the check covers the whole kernel, the producer warpgroup at its reduced budget included."""
from test_sass_rows_register_a import HGMMA_NOP, HGMMA_REG_A, LOCAL
from test_sass_wgmma_pipeline import FULL_WAIT, MIN_HGMMA_PER_FULL_WAIT, _built_library
import re
import subprocess
from collections import defaultdict


def _halo_kernels_sass(lib, cuobjdump):
    sass = subprocess.run([cuobjdump, '-sass', lib], capture_output=True, text=True, check=True).stdout
    out = defaultdict(list)
    fn = None
    for line in sass.splitlines():
        m = re.match(r'\s*Function\s*:\s*(\S+)', line)
        if m:
            fn = m.group(1) if 'conv_tc_halo_kernel' in m.group(1) else None
        elif fn is not None:
            out[fn].append(line)
    return out


def test_halo_kernel_register_a_pipelined_without_local_memory():
    lib, cuobjdump = _built_library()
    kernels = _halo_kernels_sass(lib, cuobjdump)
    assert len(kernels) == 12, sorted(kernels)   # BN = 16 / 32 / 48 / 64 / 96 / 128, MB = 1 / 2
    bad = {}
    for fn, lines in sorted(kernels.items()):
        hgmma = [l for l in lines if 'HGMMA' in l and not HGMMA_NOP.search(l)]
        smem_a = [l.strip() for l in hgmma if not HGMMA_REG_A.search(l)]
        local = [l.strip() for l in lines if LOCAL.search(l)]
        full_waits = sum(1 for l in lines if FULL_WAIT.search(l))
        if not hgmma or smem_a or local or len(hgmma) < MIN_HGMMA_PER_FULL_WAIT * max(full_waits, 1):
            bad[fn] = {'hgmma': len(hgmma), 'full_waits': full_waits, 'a_from_smem': smem_a[:2],
                       'local_memory': local[:2]}
    assert not bad, bad
