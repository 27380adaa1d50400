"""Builds libvr_b200.so (the C-ABI CUDA library, sm_90a only) in-tree with nvcc.

``python build.py`` from this directory, or ``__graft_entry__.build()`` from the repo root.  nvcc
cross-compiles without a GPU.  Objects are rebuilt only when their sources are newer.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(HERE, 'build')
LIB = os.path.join(HERE, 'libvr_b200.so')
SOURCES = ['api.cu', 'engine.cu', 'conv_simt.cu', 'conv_tc.cu', 'conv_tc_rows.cu', 'conv_tc_halo.cu', 'elementwise.cu', 'lstm.cu', 'fft.cu', 'resample.cu', 'flac.cu', 'flac_encode.cu', 'mp3.cu', 'aac.cu', 'vorbis.cu', 'bsseval.cu', 'wiener.cu']
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
         '-Xcompiler', '-fPIC', '-Xcompiler', '-fvisibility=hidden', '--expt-relaxed-constexpr']


def _newest_header():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.h', '.cuh'))]
    hs.append(os.path.join(HERE, '..', 'include', 'vr_b200.h'))
    return max(os.path.getmtime(h) for h in hs)


def build(verbose=False, force=False):
    global OBJ, LIB
    extra = os.environ.get('VR_BUILD_FLAGS', '').split()
    if os.environ.get('VR_BUILD_TAG'):
        OBJ = os.path.join(HERE, 'build_' + os.environ['VR_BUILD_TAG'])
        LIB = os.path.join(HERE, 'libvr_b200_%s.so' % os.environ['VR_BUILD_TAG'])
    os.makedirs(OBJ, exist_ok=True)
    hdr = _newest_header()
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src.replace('.cu', '.o'))
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr):
            jobs.append((s, o))

    def cc(job):
        s, o = job
        cmd = [NVCC] + FLAGS + extra + ['-c', s, '-o', o]
        if verbose:
            cmd += ['-Xptxas', '-v']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed for %s:\n%s\n%s' % (s, r.stdout, r.stderr))
        return r.stderr

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        logs = list(ex.map(cc, jobs))
    if verbose:
        for lg in logs:
            print(lg)
    objs = [os.path.join(OBJ, s.replace('.cu', '.o')) for s in SOURCES]
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC, '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a']
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('link failed:\n%s\n%s' % (r.stdout, r.stderr))
    return LIB


if __name__ == '__main__':
    print(build(verbose='-v' in sys.argv, force='-f' in sys.argv))
