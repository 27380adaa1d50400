"""The row and halo convolutions store their output with 128-bit or 64-bit global stores (no GPU needed).

epilogue_store (csrc/tc_common.cuh) transposes each quad's channel pairs so that every lane writes 8 consecutive
channels of a pixel per plane with one 16-byte store (`STG.E.128`), where epilogue_pair writes 4 bytes per channel pair.
Two kinds of variant have no registers to spare for those transposes (DESIGN 5.2, 5.7): the row kernel with the fused
upsample and the halo kernel at BN = 128, MB = 2.  They store through epilogue_pixel8, which swaps one channel pair
between neighbouring lanes and writes 4 channels per lane and plane with one 8-byte store (`STG.E.64`); the row kernel
with the fused upsample at BN = 16 measured slower that way and keeps epilogue_pair's 4-byte stores.  This reads the
SASS of the built library and checks that the consumer code of every row and halo instantiation holds the stores of its
kind, and no local memory."""
from test_sass_halo_register_a import _halo_kernels_sass
from test_sass_rows_register_a import LOCAL, _rows_kernels_sass
from test_sass_wgmma_pipeline import _built_library

STG128 = 'STG.E.128'
STG64 = 'STG.E.64'
PIXEL8 = ('conv_tc_halo_kernelILi128ELi2E',)
PAIRS = ('conv_tc_rows_kernelILi16ELb1E',)   # measured slower with 8-byte stores: epilogue_pair


def _consumer(lines):
    """the consumer code: everything from setmaxnreg.inc on, where the kernel has one"""
    alloc = [i for i, l in enumerate(lines) if 'USETMAXREG.TRY_ALLOC' in l]
    return lines[alloc[0]:] if alloc else lines


def test_row_and_halo_kernels_store_whole_sectors():
    lib, cuobjdump = _built_library()
    kernels = {**_rows_kernels_sass(lib, cuobjdump), **_halo_kernels_sass(lib, cuobjdump)}
    assert len(kernels) == 18, sorted(kernels)   # 6 row and 12 halo instantiations
    bad = {}
    for fn, lines in sorted(kernels.items()):
        code = _consumer(lines)
        stg128 = sum(1 for l in code if STG128 in l)
        stg64 = sum(1 for l in code if STG64 in l)
        local = [l.strip() for l in code if LOCAL.search(l)]
        pairs = any(k in fn for k in PAIRS)
        pixel8 = 'Lb1E' in fn and not pairs or any(k in fn for k in PIXEL8)
        ok = stg128 == 0 and stg64 == 0 if pairs else (stg64 > 0 and stg128 == 0) if pixel8 else stg128 > 0
        if local or not ok:
            bad[fn] = {'STG.E.128': stg128, 'STG.E.64': stg64, 'pixel8': pixel8, 'pairs': pairs, 'local_memory': local[:2]}
    assert not bad, bad
