# -*- coding: utf-8 -*-
"""CPU test of the compiled conv kernels: ptxas issues the wgmmas of every conv_umma_kernel / stem4_kernel instantiation as a pipeline.

When ptxas cannot pipeline a kernel's wgmmas it serialises them: every HGMMA is followed by a full wait on the wgmma group
(WARPGROUP.DEPBAR.LE gsb0, 0x0), so each MMA waits for the previous one to finish.  Pipelined, the full waits are only the ones the
source asks for.  conv_umma.cu is compiled for sm_90a, as build.py compiles it and with the LFD_B200_TRACE hooks (so that trace cycles
describe the kernel that runs), and the SASS of every instantiation is counted.  No GPU is needed; without nvcc the test is skipped."""
import importlib.util
import os
import re
import subprocess
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, 'lfd-a-light-and-fast-detector_b200')

MODE_FLAT, MODE_3X3S1, MODE_3X3S2, MODE_1X1S2, MODE_STEM = 0, 1, 2, 3, 4
# the output widths umma_conv_launch instantiates per mode
COUTS = {MODE_FLAT: (16, 32, 64, 128), MODE_3X3S1: (32, 64, 128), MODE_3X3S2: (32, 64, 128), MODE_1X1S2: (16, 32, 64, 128),
         MODE_STEM: (16, 32, 64)}
# Full waits the source asks for: conv_umma_kernel waits once per channel chunk for its main MMAs (plus the fused shortcut's) and once
# in each of the four tail widths (16 / 32 / 64 / 128) of a kernel without the shortcut; stem4_kernel waits for stem0, stem1, stem2 and
# the stem3 tail.
WAITS_CONV, WAITS_CONV_DS, WAITS_STEM4 = 5, 1, 4

_CONV = re.compile(r'_ZN3lfd16conv_umma_kernelILi(\d)ELi(\d+)ELb([01])ELb([01])ELb([01])EEEvNS_14UmmaConvParamsE')
_STEM4 = re.compile(r'_ZN3lfd12stem4_kernelILb([01])ELb([01])EEEvNS_14UmmaConvParamsE')


def _build_module():
    spec = importlib.util.spec_from_file_location('lfd_build', os.path.join(PKG, 'build.py'))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    return b


def _sass_counts(obj, cuobjdump):
    """{kernel name: (HGMMA count, full-wait count)} of every function in the object file"""
    sass = subprocess.run([cuobjdump, '-sass', obj], check=True, capture_output=True, text=True).stdout
    counts, name = {}, None
    for line in sass.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            name = m.group(1)
            counts[name] = [0, 0]
        elif name and 'HGMMA' in line:
            counts[name][0] += 1
        elif name and 'WARPGROUP.DEPBAR.LE gsb0, 0x0' in line:
            counts[name][1] += 1
    return {k: tuple(v) for k, v in counts.items()}


@pytest.fixture(scope='module')
def sass():
    b = _build_module()
    cuobjdump = os.path.join(os.path.dirname(b.NVCC), 'cuobjdump')
    if not (os.path.exists(b.NVCC) and os.path.exists(cuobjdump)):
        pytest.skip('nvcc / cuobjdump not found at %s' % os.path.dirname(b.NVCC))
    flags = [f for f in b.FLAGS if f != '-DLFD_B200_TRACE']
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        procs = {}
        for variant, extra in (('plain', []), ('trace', ['-DLFD_B200_TRACE'])):
            obj = os.path.join(tmp, 'conv_umma_%s.o' % variant)
            cmd = [b.NVCC] + flags + extra + ['-c', os.path.join(b.CSRC, 'conv_umma.cu'), '-o', obj]
            procs[variant] = (obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
        for variant, (obj, p) in procs.items():
            log = p.communicate()[0].decode()
            assert p.returncode == 0, log
            out[variant] = _sass_counts(obj, cuobjdump)
    return out


def _expected_conv():
    return {(mode, cout, f16, ext, ds) for mode, couts in COUTS.items() for cout in couts for f16 in (0, 1) for ext in (0, 1)
            for ds in ((0, 1) if mode == MODE_3X3S2 else (0,))}


@pytest.mark.parametrize('variant', ['plain', 'trace'])
def test_every_conv_instantiation_pipelines_its_wgmmas(sass, variant):
    counts = sass[variant]
    found = {}
    for name, c in counts.items():
        m = _CONV.fullmatch(name)
        if m:
            found[tuple(int(g) for g in m.groups())] = c
    assert set(found) == _expected_conv(), set(found) ^ _expected_conv()
    bad = {}
    for key, (hgmma, waits) in sorted(found.items()):
        allowed = WAITS_CONV_DS if key[4] else WAITS_CONV
        if hgmma == 0 or waits > allowed:
            bad[key] = (hgmma, waits, allowed)
    assert not bad, 'conv_umma_kernel<MODE, COUT, F16, EXT, DS>: (HGMMA, full waits, designed waits) %s' % bad


@pytest.mark.parametrize('variant', ['plain', 'trace'])
def test_fused_stem_pipelines_its_wgmmas(sass, variant):
    found = {tuple(int(g) for g in _STEM4.fullmatch(n).groups()): c for n, c in sass[variant].items() if _STEM4.fullmatch(n)}
    assert set(found) == {(f16, ext) for f16 in (0, 1) for ext in (0, 1)}
    for key, (hgmma, waits) in found.items():
        assert hgmma > 0 and waits <= WAITS_STEM4, ('stem4_kernel', key, hgmma, waits)


def test_build_guard_rejects_serialised_wgmmas():
    b = _build_module()
    conv = '_ZN3lfd16conv_umma_kernelILi1ELi64ELb0ELb0ELb0EEEvNS_14UmmaConvParamsE'
    msg = ("ptxas info    : (%s) Potential Performance Loss: wgmma.mma_async instructions are serialized due to %s in the function '%s'")
    b._check_stack_frames('ptxas info    : (C7519) warpgroup.arrive is injected in around line 1 by compiler to allow use of registers '
                          "in GMMA in function '%s'" % conv)
    for code, why in (('C7511', 'insufficient register resources for the wgmma pipeline'),
                      ('C7512', 'insufficient register resources for the function'),
                      ('C7520', 'program dependence on compiler-inserted WG.AR in divergent path')):
        with pytest.raises(RuntimeError):
            b._check_stack_frames(msg % (code, why, conv))
        with pytest.raises(RuntimeError):
            b._check_stack_frames(msg % (code, why, '_ZN3lfd12stem4_kernelILb0ELb0EEEvNS_14UmmaConvParamsE'))
        b._check_stack_frames(msg % (code, why, '_ZN3lfd17wgrad_umma_kernelILi0ELi64EEEvNS0_11WgradParamsE'))   # not guarded
