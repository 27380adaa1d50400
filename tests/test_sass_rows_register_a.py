"""The row-streaming convolution reads its A operand from registers and keeps everything in registers (no GPU needed).

Each input row of conv_tc_rows_kernel feeds up to three output rows, three products each.  The kernel loads a row's A
fragments once per kw tap with ldmatrix and every wgmma of that row takes them from registers (`HGMMA ... R, R,
gdesc`), instead of re-reading the same tile from shared memory per wgmma (`HGMMA ... R, gdesc, gdesc`).  Holding the
fragments next to the accumulators needs the registers that setmaxnreg moves to the consumer warpgroups; if they do not
fit, ptxas spills to local memory (STL / LDL).  This reads the SASS of the built library and checks that every HGMMA
takes A from registers, and that the consumer code has no local-memory access: the whole kernel without the fused
upsample, and with it everything from the consumers' `USETMAXREG.TRY_ALLOC` on (the producer warps are laid out
before it; at 72 registers the interpolation warps keep one 4-byte value of their per-tile set-up in local memory).
If ptxas ever places producer code after that point, the check covers it too and can only become stricter.

setmaxnreg.inc takes registers only from what the block was launched with: the fused-upsample variants must launch
with the register count the budget in conv_tc_rows.cu assumes (kUpLaunchRegs), or the consumers wait forever."""
import os
import re
import subprocess
from collections import defaultdict

from conftest import PKG
from test_sass_wgmma_pipeline import _built_library

HGMMA_REG_A = re.compile(r'HGMMA\.\S+\s+R\d+\s*,\s*R\d+\s*,\s*gdesc\[')
# ptxas places an HGMMA without operands or destination (`HGMMA.64x8x16.F16 RZ, gdesc[URZ], RZ, !UPT`) where a
# commit group can be empty: it computes nothing
HGMMA_NOP = re.compile(r'HGMMA\.\S+\s+RZ\s*,')
LOCAL = re.compile(r'\b(STL|LDL)(\.\S+)?\s')


def _rows_kernels_sass(lib, cuobjdump):
    """{mangled conv_tc_rows_kernel name: list of its SASS lines}"""
    sass = subprocess.run([cuobjdump, '-sass', lib], capture_output=True, text=True, check=True).stdout
    out = defaultdict(list)
    fn = None
    for line in sass.splitlines():
        m = re.match(r'\s*Function\s*:\s*(\S+)', line)
        if m:
            fn = m.group(1) if 'conv_tc_rows_kernel' in m.group(1) else None
        elif fn is not None:
            out[fn].append(line)
    return out


def test_row_kernel_wgmma_take_a_from_registers_without_local_memory():
    lib, cuobjdump = _built_library()
    kernels = _rows_kernels_sass(lib, cuobjdump)
    assert len(kernels) == 6, sorted(kernels)   # BN = 16 / 32 / 64, with and without the fused upsample
    bad = {}
    for fn, lines in sorted(kernels.items()):
        hgmma = [l for l in lines if 'HGMMA' in l and not HGMMA_NOP.search(l)]
        smem_a = [l.strip() for l in hgmma if not HGMMA_REG_A.search(l)]
        alloc = [i for i, l in enumerate(lines) if 'USETMAXREG.TRY_ALLOC' in l]
        up = 'Lb1E' in fn
        if up and len(alloc) != 1:
            bad[fn] = {'setmaxnreg.inc sites': len(alloc)}
            continue
        first_hgmma = next(i for i, l in enumerate(lines) if 'HGMMA' in l) if hgmma else 0
        start = alloc[0] if up else 0
        local = [l.strip() for l in lines[start:] if LOCAL.search(l)]
        if start > first_hgmma:
            local.append('HGMMA before the consumer branch: layout not understood')
        if not hgmma or smem_a or local:
            bad[fn] = {'hgmma': len(hgmma), 'a_from_smem': smem_a[:2], 'local_memory': local[:2]}
    assert not bad, bad


def test_fused_upsample_variants_launch_with_the_register_budget_they_assume():
    lib, cuobjdump = _built_library()
    src = open(os.path.join(PKG, 'csrc', 'conv_tc_rows.cu')).read()
    launch = int(re.search(r'kUpLaunchRegs\s*=\s*(\d+)', src).group(1))
    usage = subprocess.run([cuobjdump, '-res-usage', lib], capture_output=True, text=True, check=True).stdout
    regs = dict(re.findall(r'Function (\S*conv_tc_rows_kernel\S*Lb1E\S*):\s*\n\s*REG:(\d+)', usage))
    assert len(regs) == 3, regs
    assert all(int(r) >= launch for r in regs.values()), (launch, regs)
