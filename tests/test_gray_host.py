# -*- coding: utf-8 -*-
"""Gray (1-channel) models on the host: the planners emit STEM0 / STEM4 ops with Cin = 1 whose packed parameters are, byte for byte, those
of the 3-channel twin with stem weights [W1, 0, 0] (tests/gray_models.py); the training planner plans a gray stem; the input transform of a
gray model; model files of gray plans through lfd_engine_open; and the stem kernels, compiled with the gray loaders, still pipeline their
wgmmas without a stack frame."""
import ctypes as C
import os
import re
import struct
import subprocess
import tempfile

import pytest
import torch

from gray_models import gray_pair
from lfd import _native as nat
from lfd._engine import InferencePlan, PostPlan, pack_stem_weight
from lfd._train import TrainPlan
from lfd.data_pipeline.augmentation import (BGR2RGB, Compose, InputTransform, Normalize, caffe_imagenet_normalize, input_transform_of,
                                            simple_normalize, simple_widerface_val_pipeline, standard_normalize)
from test_conv_sass import WAITS_CONV, WAITS_STEM4, _build_module, _sass_counts
from test_engine_file_host import HEADER, LFD_ERR_INVALID, open_engine, op_at, refused, resign

CPU = torch.device('cpu')


def plans(name, N=2, H=200, W=264, **kw):
    gray, twin = gray_pair(name)
    return (InferencePlan(gray, N, H, W, CPU, create_native=False, **kw), InferencePlan(twin, N, H, W, CPU, create_native=False, **kw))


def assert_same_plan(g, t):
    """The gray plan is the twin's with Cin = 1 on its image op: same ops, same workspace, same packed parameters."""
    assert len(g._ops) == len(t._ops) and g.workspace_bytes == t.workspace_bytes and g.P == t.P
    assert g._ops[0]['Cin'] == 1 and t._ops[0]['Cin'] == 3
    assert all(o['Cin'] != 1 for o in g._ops[1:])
    for a, b in zip(g._op_array, t._op_array):
        for f, typ in nat.Op._fields_:
            if f != 'Cin' and typ is not C.c_void_p:        # (pointers: into each plan's own parameter buffers, compared below)
                assert repr(getattr(a, f)) == repr(getattr(b, f)) or list(getattr(a, f)) == list(getattr(b, f)), f
    assert torch.equal(g.params_bf16, t.params_bf16) and torch.equal(g.params_f32, t.params_f32)


@pytest.mark.parametrize('name,fuse,kind,cout,tail', [
    ('WIDERFACE_S', True, nat.OP_STEM4, 64, 64),        # the 'faster' stem as one kernel
    ('WIDERFACE_S', False, nat.OP_STEM0, 64, 64),       # ... and as STEM0 + tail, CONV + tail
    ('WIDERFACE_XS', False, nat.OP_STEM0, 32, 32),
    ('WIDERFACE_L', None, nat.OP_STEM0, 64, 64),        # 'fast' stem
    ('TL_S', None, nat.OP_STEM0, 48, 48),                # the 48-wide 'fast' stem (conv_umma_c48_kernel)
    ('TEST_FASTEST', None, nat.OP_STEM0, 16, 0),        # 'fastest' stem: no tail
])
def test_inference_planner_emits_gray_stem_ops(name, fuse, kind, cout, tail):
    g, t = plans(name, fuse_stem=fuse)
    op = g._ops[0]
    assert (op['kind'], op['Cin'], op['Cout'], op.get('tail_cout', 0)) == (kind, 1, cout, tail), op
    assert_same_plan(g, t)


def test_pack_stem_weight_puts_the_gray_channel_in_the_channel_0_lanes():
    w1 = torch.randn(32, 1, 3, 3)
    w3 = torch.cat([w1, torch.zeros(32, 2, 3, 3)], 1)
    assert torch.equal(pack_stem_weight(w1).view(torch.int16), pack_stem_weight(w3).view(torch.int16))
    full = pack_stem_weight(w1, torch.float32).reshape(3, 2, 32, 2, 4)     # [kh][kc][n][pixel][channel]
    assert bool((full[..., 1:] == 0).all()) and float(full[..., 0].abs().sum()) > 0


def test_other_channel_counts_stay_refused():
    gray, _ = gray_pair('WIDERFACE_L')
    two = torch.nn.Conv2d(2, 64, 3, 2, 1, bias=False)
    gray._backbone._stem[0] = two
    with pytest.raises(NotImplementedError, match='1-channel'):
        InferencePlan(gray, 1, 64, 64, CPU, create_native=False)


@pytest.mark.parametrize('frozen', [None, 1])
def test_training_planner_plans_a_gray_stem(frozen):
    gray, twin = gray_pair('WIDERFACE_L')
    for m in (gray, twin):
        if frozen:
            m._backbone._frozen_stages = frozen
        m.train()
    g = TrainPlan(gray, 2, 128, 160, CPU, create_native=False)
    t = TrainPlan(twin, 2, 128, 160, CPU, create_native=False)
    assert g.in_channels == 1 and t.in_channels == 3
    assert [o['kind'] for o in g.fwd_ops] == [o['kind'] for o in t.fwd_ops]
    assert [o['kind'] for o in g.bwd_ops] == [o['kind'] for o in t.bwd_ops]
    assert g.workspace_bytes == t.workspace_bytes
    if frozen:          # the frozen prefix runs the gray stem on the inference kernels: no stem op of the training kind, no stem gradient
        infer = [o for o in g.fwd_ops if o['kind'] == nat.TOP_INFER]
        assert infer and not any(o['kind'] in (nat.TOP_STEM0, nat.TOP_WGRAD_STEM) for o in g.fwd_ops + g.bwd_ops)
        stems = [o for o in g.fwd_ops if o['kind'] == nat.TOP_INFER and o['Cin'] == 1]
        assert len(stems) == 1
    else:
        stem0 = [o for o in g.fwd_ops if o['kind'] == nat.TOP_STEM0]
        wstem = [o for o in g.bwd_ops if o['kind'] == nat.TOP_WGRAD_STEM]
        assert len(stem0) == 1 and stem0[0]['Cin'] == 1 and len(wstem) == 1 and wstem[0]['Cin'] == 1
        # the stem's weight packing and its gradient's unpacking with Cin = 1; the gradient staging keeps the 32 rows of the wgmma path
        conv = gray._backbone._stem[0]
        pack = [d for d in g._pack.items if d.kind == nat.PACK_STEM]
        unpack = [d for d in g._unpack.items if d.kind == nat.UNPACK_CONV and d.Cin == 1]
        assert len(pack) == 1 and (pack[0].Cin, pack[0].Cout, pack[0].n) == (1, 64, 3 * 2 * 64 * 8)
        assert len(unpack) == 1 and (unpack[0].kk, unpack[0].Cout, unpack[0].n) == (9, 64, 64 * 9)
        assert g._sizes[g._gstage[id(conv.weight)]] == 32 * 64 * 4


# ------------------------------------------------------------------------------------------------------------------ input transform
def test_input_transform_of_a_gray_model():
    m, s = simple_normalize.constants()
    assert input_transform_of(None, channels=1) is None
    t = input_transform_of(simple_widerface_val_pipeline, channels=1)
    assert t == InputTransform(False, (float(m[0]),) * 3, (float(s[0]),) * 3)
    one = Normalize(mean=(0.25,), std=(0.125,), max_pixel_value=255.0, p=1.0)
    m1, s1 = one.constants()
    assert input_transform_of(Compose([one]), channels=1) == InputTransform(False, (float(m1[0]),) * 3, (float(s1[0]),) * 3)
    assert input_transform_of(InputTransform(False, (3.0,) * 3, (0.5,) * 3), channels=1) == InputTransform(False, (3.0,) * 3, (0.5,) * 3)
    for bad in (Compose([BGR2RGB()]), Compose([BGR2RGB(), simple_normalize]), Compose([standard_normalize]), Compose([caffe_imagenet_normalize]),
                InputTransform(True, (1.0,) * 3, (1.0,) * 3), InputTransform(False, (1.0, 2.0, 1.0), (1.0,) * 3)):
        with pytest.raises(ValueError):
            input_transform_of(bad, channels=1)
    # the 3-channel lowering is unchanged
    assert input_transform_of(Compose([standard_normalize])).mean == tuple(float(v) for v in standard_normalize.constants()[0])


def test_set_input_transform_checks_the_model_kind():
    gray, twin = gray_pair('WIDERFACE_XS')
    with pytest.raises(ValueError):
        gray.set_input_transform(Compose([standard_normalize]))
    twin.set_input_transform(Compose([standard_normalize]))
    gray.set_input_transform(simple_widerface_val_pipeline)
    assert len(set(gray.input_transform.mean)) == 1


# ------------------------------------------------------------------------------------------------------------------ model files
@pytest.fixture(scope='module')
def gray_file():
    gray, _ = gray_pair('WIDERFACE_S')
    gray.set_input_transform(simple_widerface_val_pipeline)
    plan = InferencePlan(gray, 1, 128, 160, CPU, create_native=False, fuse_stem=True, input_transform=gray.input_transform)
    post = PostPlan(gray._post_cfg(1, plan.level_sizes, 0.3, 0.4, False), CPU)
    return plan, plan.model_file_bytes(post)


def test_engine_opens_a_gray_file(gray_file):
    plan, data = gray_file
    rc, e, msg = open_engine(data)
    assert rc == 0, msg
    try:
        got, src, level = nat.Op(), C.c_int32(), C.c_int32()
        nat.check(nat.lib().lfd_engine_op(e, 0, C.byref(got), C.byref(src), C.byref(level)))
        assert (got.kind, got.Cin) == (nat.OP_STEM4, 1)
    finally:
        nat.lib().lfd_engine_close(e)


def test_engine_refuses_a_gray_file_with_another_channel_count_or_a_swap(gray_file):
    _, data = gray_file
    for cin in (2, 0, 4):
        b = bytearray(data)
        struct.pack_into('<i', b, op_at(data, 0) + nat.Op.Cin.offset, cin)
        msg = refused(resign(b), LFD_ERR_INVALID, 'op 0')
        assert 'channels' in msg or 'Cin' in msg, msg
    # in_swap_rb = 1 on op 0 and in the plan section (which have to agree): the gray image op refuses it
    b = bytearray(data)
    struct.pack_into('<i', b, op_at(data, 0) + nat.Op.in_swap_rb.offset, 1)
    struct.pack_into('<i', b, HEADER + 56, 1)
    assert 'gray' in refused(resign(b), LFD_ERR_INVALID, 'input transform')
    # unequal constants
    b = bytearray(data)
    mean = struct.unpack_from('<3f', data, HEADER + 60)
    struct.pack_into('<f', b, op_at(data, 0) + nat.Op.in_mean.offset + 4, mean[1] + 1.0)
    struct.pack_into('<f', b, HEADER + 64, mean[1] + 1.0)
    assert 'gray' in refused(resign(b), LFD_ERR_INVALID, 'input transform')


# ------------------------------------------------------------------------------------------------------------------ compiled kernels
_STEM_CONV = re.compile(r'_ZN3lfd16conv_umma_kernelILi4ELi(\d+)ELb([01])ELb([01])ELb0EEEvNS_14UmmaConvParamsE')
_STEM_C48 = re.compile(r'_ZN3lfd20conv_umma_c48_kernelILi4ELb([01])ELb([01])ELb0EEEvNS_14UmmaConvParamsE')
_STEM4 = re.compile(r'_ZN3lfd12stem4_kernelILb([01])ELb([01])EEEvNS_14UmmaConvParamsE')


def test_every_stem_instantiation_pipelines_its_wgmmas_without_a_stack_frame():
    """The stem producers specialise gray and BGR at compile time (stem4_kernel through the shared decoder of image.cuh, the MODE_STEM
    producer in its own loader): conv_umma.cu as build.py compiles it, with ptxas -v.  Every stem instantiation (conv_umma_kernel MODE_STEM 16 / 32 / 64,
    conv_umma_c48_kernel MODE_STEM, stem4_kernel) has no stack frame and keeps its wgmma pipeline."""
    b = _build_module()
    cuobjdump = os.path.join(os.path.dirname(b.NVCC), 'cuobjdump')
    if not (os.path.exists(b.NVCC) and os.path.exists(cuobjdump)):
        pytest.skip('nvcc / cuobjdump not found at %s' % os.path.dirname(b.NVCC))
    flags = [f for f in b.FLAGS if f != '-DLFD_B200_TRACE']
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, 'conv_umma.o')
        p = subprocess.run([b.NVCC] + flags + ['-Xptxas', '-v', '-c', os.path.join(b.CSRC, 'conv_umma.cu'), '-o', obj],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        log = p.stdout.decode()
        assert p.returncode == 0, log
        b._check_stack_frames(log, limit=0)
        counts = _sass_counts(obj, cuobjdump)
    frames, name = {}, None
    for line in log.splitlines():
        m = re.search(r'Function properties for (\S+)', line)
        if m:
            name = m.group(1)
        m = re.search(r'(\d+) bytes stack frame', line)
        if m and name:
            frames[name] = int(m.group(1))
    stems = {n: c for n, c in counts.items() if _STEM_CONV.fullmatch(n) or _STEM_C48.fullmatch(n) or _STEM4.fullmatch(n)}
    assert len([n for n in stems if _STEM_CONV.fullmatch(n)]) == 3 * 2 * 2
    assert len([n for n in stems if _STEM_C48.fullmatch(n)]) == 2 * 2 and len([n for n in stems if _STEM4.fullmatch(n)]) == 2 * 2
    for n, (hgmma, waits) in stems.items():
        assert frames.get(n) == 0, (n, frames.get(n))
        assert hgmma > 0 and waits <= (WAITS_STEM4 if _STEM4.fullmatch(n) else WAITS_CONV), (n, hgmma, waits)
