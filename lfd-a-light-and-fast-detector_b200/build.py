# -*- coding: utf-8 -*-
"""Builds liblfd_b200.so (sm_90a, H100) in-tree with nvcc.  No GPU is needed to compile.

    python build.py [--force] [--verbose]

LFD_B200_TRACE=1 compiles the clock64() per-role hooks of the convolution kernel in (tests/debug_trace.py) and
LFD_B200_TIMELINE=1 the per-launch %globaltimer stamps (tests/debug_timeline.py); both are absent from the normal build.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.environ.get('LFD_B200_OUT') or os.path.join(HERE, 'liblfd_b200.so')      # LFD_B200_OUT / LFD_B200_EXTRA_FLAGS: tuning experiments only
SOURCES = ['api.cu', 'conv_umma.cu', 'conv_simt.cu', 'postprocess.cu', 'losses.cu', 'train.cu', 'wgrad_umma.cu', 'input.cu']
HEADERS = ['ptx.cuh', 'image.cuh', 'conv_common.cuh', 'kernels.cuh', 'train.cuh', os.path.join('..', '..', 'include', 'lfd_b200.h')]
INCLUDE = os.path.join(os.path.dirname(HERE), 'include')
# the C program that runs a model file through the library and cudart alone (include/lfd_b200.h, lfd_engine_*), built next to the library
EXAMPLE = os.path.join(os.path.dirname(HERE), 'examples', 'lfd_detect.c')
EXAMPLE_OUT = os.path.join(os.path.dirname(OUT), 'lfd_detect')
NVCC = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a']
FLAGS = ARCH + ['-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC',
                '--expt-relaxed-constexpr'] + (['-DLFD_B200_TRACE'] if os.environ.get('LFD_B200_TRACE') else []) + \
        (['-DLFD_B200_TIMELINE'] if os.environ.get('LFD_B200_TIMELINE') else []) + os.environ.get('LFD_B200_EXTRA_FLAGS', '').split()


def _stale(out, deps):
    return not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps)


# kernels whose per-thread state must stay in registers (the soft-NMS kernel runs one iteration per candidate: a spill is paid K times)
# (kernel names are matched by substring: conv_umma_solo_kernel is not covered by conv_umma_kernel and is listed on its own)
_STACK_GUARDED = ('conv_umma_kernel', 'conv_umma_c48_kernel', 'conv_umma_solo_kernel', 'stem4_kernel', 'soft_nms_kernel')
# kernels whose wgmmas must be pipelined: every instantiation, no exemptions
_WGMMA_GUARDED = ('conv_umma_kernel', 'conv_umma_c48_kernel', 'conv_umma_solo_kernel', 'stem4_kernel')
_PTXAS_VERBOSE = ('conv_umma.cu', 'postprocess.cu')


def _check_stack_frames(ptxas_log, limit=64):
    """The warp-specialised conv kernel keeps its accumulators and role state in registers; a large stack frame means a lambda
    was not inlined or an array went to local memory, which slows the kernel severalfold.  Fail the build instead.

    Also fail it when ptxas serialised the wgmmas of a conv kernel (C7511 / C7512: too few registers for the wgmma pipeline; C7520:
    a compiler-inserted warpgroup.arrive on a divergent path): every MMA then waits for the previous one to finish, and which
    instantiations it hits changes with unrelated edits."""
    import re
    name = None
    for line in ptxas_log.splitlines():
        m = re.search(r'Function properties for (\S+)', line)
        if m:
            name = m.group(1)
        m = re.search(r'(\d+) bytes stack frame', line)
        if m and name and any(k in name for k in _STACK_GUARDED) and int(m.group(1)) > limit:
            raise RuntimeError('%s has a %s-byte stack frame (limit %d): registers went to local memory' % (name, m.group(1), limit))
        m = re.search(r'\((C75\d\d)\).*wgmma\.mma_async instructions are serialized.*\'(\S+)\'', line)
        if m and any(k in m.group(2) for k in _WGMMA_GUARDED):
            raise RuntimeError('ptxas serialised the wgmma instructions of %s (%s):\n%s' % (m.group(2), m.group(1), line))


def build(force=False, verbose=False):
    """The library, then the example program; each is rebuilt only when its own inputs changed."""
    build_library(force, verbose)
    build_example(force)
    return OUT


def build_library(force=False, verbose=False):
    if not force and not _stale(OUT, [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]):
        return OUT
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(CSRC, s.replace('.cu', '.o')) if not os.environ.get('LFD_B200_OUT') else os.path.join('/tmp', os.path.basename(OUT) + '.' + s.replace('.cu', '.o'))
        # conv_umma.cu and postprocess.cu are always compiled with ptxas -v: see _check_stack_frames
        cmd = [NVCC] + FLAGS + (['-Xptxas', '-v'] if (verbose or s in _PTXAS_VERBOSE) else []) + ['-c', os.path.join(CSRC, s), '-o', o]
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(o)
    for s, p in procs:
        out = p.communicate()[0].decode()
        if p.returncode != 0:
            raise RuntimeError('nvcc failed on %s:\n%s' % (s, out))
        if s in _PTXAS_VERBOSE:
            _check_stack_frames(out)
            if not verbose:
                out = '\n'.join(l for l in out.splitlines() if 'ptxas info' not in l and 'bytes stack frame' not in l)
        if verbose or out.strip():
            sys.stderr.write(out)
    subprocess.check_call([NVCC, '-shared', '-o', OUT] + objs + ARCH + ['-lcudart'])
    return OUT


def build_example(force=False):
    """examples/lfd_detect.c, host code only: linked against the library by its file name (found next to the program at run time) and
    the shared cudart the library uses."""
    if not force and not _stale(EXAMPLE_OUT, [EXAMPLE, OUT, os.path.join(INCLUDE, 'lfd_b200.h'), os.path.abspath(__file__)]):
        return EXAMPLE_OUT
    subprocess.check_call([NVCC] + ARCH + ['-O2', '-I', INCLUDE, EXAMPLE, '-o', EXAMPLE_OUT, '-L', os.path.dirname(OUT), '-l:' + os.path.basename(OUT),
                           '-cudart', 'shared', '-Xlinker', '-rpath,$ORIGIN'])
    return EXAMPLE_OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
