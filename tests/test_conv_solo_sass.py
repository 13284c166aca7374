# -*- coding: utf-8 -*-
"""CPU tests of conv_umma_solo_kernel, the 64-channel 3x3/s1 conv whose two consumer warpgroups take whole tiles and alternate on the
tensor cores: ptxas pipelines its wgmmas (one full wait, for the main chain) in the normal and the LFD_B200_TRACE build, build.py
guards it, and the configurator picks it for the geometries it was made for and no others."""
import os
import subprocess
import tempfile
import re

import pytest

from test_conv_sass import _build_module, _sass_counts

_SOLO = re.compile(r'_ZN3lfd21conv_umma_solo_kernelILb([01])ELb([01])EEEvNS_14UmmaConvParamsE')
HGMMA_SOLO, WAITS_SOLO = 72, 1   # 4 k16 steps x 9 taps x 2 m64 blocks; one wait for the whole chain


@pytest.fixture(scope='module')
def solo_sass():
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
            cmd = [b.NVCC] + flags + extra + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'conv_umma.cu'), '-o', obj]
            procs[variant] = (obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT))
        for variant, (obj, p) in procs.items():
            log = p.communicate()[0].decode()
            assert p.returncode == 0, log
            b._check_stack_frames(log)         # no stack frame, no serialised wgmmas
            out[variant] = _sass_counts(obj, cuobjdump)
    return out


@pytest.mark.parametrize('variant', ['plain', 'trace'])
def test_solo_kernel_pipelines_its_wgmmas(solo_sass, variant):
    found = {tuple(int(v) for v in _SOLO.fullmatch(n).groups()): c for n, c in solo_sass[variant].items() if _SOLO.fullmatch(n)}
    assert set(found) == {(f16, ext) for f16 in (0, 1) for ext in (0, 1)}, found
    for key, (hgmma, waits) in found.items():
        assert hgmma == HGMMA_SOLO and waits <= WAITS_SOLO, ('conv_umma_solo_kernel', key, hgmma, waits)


def test_build_guards_the_solo_kernel():
    b = _build_module()
    name = '_ZN3lfd21conv_umma_solo_kernelILb0ELb0EEEvNS_14UmmaConvParamsE'
    for code, why in (('C7511', 'insufficient register resources for the wgmma pipeline'),
                      ('C7512', 'insufficient register resources for the function'),
                      ('C7520', 'program dependence on compiler-inserted WG.AR in divergent path')):
        with pytest.raises(RuntimeError):
            b._check_stack_frames("ptxas info    : (%s) Potential Performance Loss: wgmma.mma_async instructions are serialized due to %s "
                                  "in the function '%s'" % (code, why, name))
    with pytest.raises(RuntimeError):
        b._check_stack_frames('ptxas info    : Function properties for %s\n    256 bytes stack frame, 0 bytes spill stores' % name)


def _co(v, k, s):
    return (v + 2 * (k // 2) - k) // s + 1


# (N, H, W, Cin, Cout, k, s, tail) -> schedule on 132 SMs: solo with more tiles than CTAs.  The first three are the 64 -> 64 3x3/s1
# body convs of the WIDERFACE-S 8 x 720 x 1280 plan (stage 0 at 90 x 160: 960 tiles; stage 1 at 45 x 80: 240; stage 2 at 23 x 40: 80).
SCHEDULES = {
    (8, 90, 160, 64, 64, 3, 1, 0): 'solo',
    (8, 45, 80, 64, 64, 3, 1, 0): 'solo',
    (8, 23, 40, 64, 64, 3, 1, 0): 'shared',
    (4, 45, 88, 64, 64, 3, 1, 0): 'shared',       # 132 tiles: one per CTA
    (4, 45, 89, 64, 64, 3, 1, 0): 'solo',         # 144 tiles
    (1, 90, 160, 64, 64, 3, 1, 0): 'shared',      # 120 tiles
    (2, 90, 160, 64, 64, 3, 1, 0): 'solo',        # 240 tiles
    (8, 90, 160, 64, 64, 3, 1, 64): 'shared',     # fused tail
    (8, 90, 160, 64, 128, 3, 1, 0): 'shared',
    (8, 90, 160, 128, 64, 3, 1, 0): 'shared',
    (8, 90, 160, 32, 64, 3, 1, 0): 'shared',
    (8, 90, 160, 64, 64, 1, 1, 0): 'shared',
    (8, 180, 320, 64, 64, 3, 2, 0): 'shared',
}


def test_configurator_picks_the_solo_schedule_from_the_geometry():
    from lfd import _native as nat
    bad = {}
    for case, want in SCHEDULES.items():
        N, H, W, Cin, Cout, k, s, tail = case
        q = nat.conv_query(N, H, W, Cin, _co(H, k, s), _co(W, k, s), Cout, k, s, tail, 0)
        if q['schedule'] != want:
            bad[case] = (q['schedule'], want, q['num_tiles'])
        if want == 'solo':
            assert (q['cc'], q['weights_resident']) == (64, 1) and q['stages'] >= 3, (case, q)
    assert not bad, bad


def test_configured_cases_keep_the_shared_schedule():
    """None of the configurations test_gpu_conv_configs.py pins is a solo conv, so their (cc, weights_resident, stages) are those of
    conv_umma_kernel"""
    import test_gpu_conv_configs as t
    for case, _ in t.CASES:
        assert t._query(case)['schedule'] == 'shared', case
