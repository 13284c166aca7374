# -*- coding: utf-8 -*-
"""The input transform of the uint8 path (BGR -> RGB and any Normalize inside the stem kernels), host side: lowering of the pipelines,
the C structs and their all-zero default, where the planners put the transform and the plan caches."""
import ctypes as C

import numpy as np
import pytest
import torch

import tl_s
from helpers import synth_model
from lfd import _native as nat
from lfd._engine import InferencePlan
from lfd.data_pipeline.augmentation import (BGR2RGB, Compose, HorizontalFlip, InputTransform, Normalize, bbox_param,
                                            caffe_imagenet_normalize, input_transform_of, simple_normalize, simple_widerface_train_pipeline,
                                            simple_widerface_val_pipeline, standard_normalize, typical_coco_val_pipeline)

F32 = np.float32


def tl_val_pipeline(sample):
    """TrafficLight_train/TL_augmentation_pipeline.py: BGR2RGB + standard_normalize, the Compose picked by the sample's keys."""
    with_boxes = Compose([BGR2RGB(), standard_normalize], bbox_params=bbox_param, p=1.)
    without = Compose([BGR2RGB(), standard_normalize], p=1.)
    return with_boxes(**sample) if 'bboxes' in sample else without(**sample)


def opaque(pipeline):
    """The same pipeline as a function the lowering cannot see through: it forces the host path."""
    def run(sample):
        assert sample['image'].shape[2] == 3          # looks at the pixels, as an arbitrary host pipeline does
        return pipeline(dict(sample))
    return run


def _f32(*v):
    return tuple(float(F32(x)) for x in v)


def test_lowering_of_the_shipped_pipelines():
    assert input_transform_of(None) is None
    inv = float(F32(1) / F32(127.5))
    assert input_transform_of(simple_widerface_val_pipeline) == InputTransform(False, (127.5,) * 3, (inv,) * 3)
    assert input_transform_of(typical_coco_val_pipeline) == InputTransform(False, _f32(102.9801, 115.9465, 122.7717), (1.0, 1.0, 1.0))
    t = input_transform_of(tl_val_pipeline)
    m = np.array([0.485, 0.456, 0.406], F32) * F32(255)
    s = np.reciprocal(np.array([0.229, 0.224, 0.225], F32) * F32(255), dtype=F32)
    assert t == InputTransform(True, tuple(map(float, m)), tuple(map(float, s)))       # indexed by NETWORK channel: R, G, B
    assert input_transform_of(Compose([BGR2RGB()])) == InputTransform(True, (0.0,) * 3, (1.0,) * 3)
    assert input_transform_of(t) is t and hash(t) == hash(input_transform_of(tl_val_pipeline))
    # the loader keeps the flip in its input kernel
    assert input_transform_of(simple_widerface_train_pipeline, allow_flip=True) == input_transform_of(simple_widerface_val_pipeline)


BAD = {'flip': simple_widerface_train_pipeline,
       'normalize-not-last': Compose([simple_normalize, BGR2RGB()]),
       'opaque': opaque(simple_widerface_val_pipeline),
       'p<1': Compose([Normalize(p=0.5)])}


@pytest.mark.parametrize('name', sorted(BAD))
def test_pipelines_the_kernels_cannot_run_are_rejected(name):
    from lfd.pipeline import StreamingDetector
    model = tl_s.build_model()
    with pytest.raises(ValueError, match='stem kernels cannot run'):
        model.set_input_transform(BAD[name])
    assert model.input_transform is None
    with pytest.raises(ValueError, match='stem kernels cannot run'):      # before any device work
        StreamingDetector(model, 1, 64, 64, 0.3, 0.3, device='cpu', input_pipeline=BAD[name])


def test_structs_have_the_library_sizes_and_the_new_fields():
    L = nat.lib()
    assert L.lfd_struct_bytes(0) == C.sizeof(nat.Op) and L.lfd_struct_bytes(1) == C.sizeof(nat.Top)
    for st in (nat.Op, nat.Top):
        names = [f[0] for f in st._fields_]
        assert names[-4:] == ['in_swap_rb', 'in_mean', 'in_scale', 'pad2_']
        o = st()
        nat.set_input_transform(o, None)
        assert bytes(o) == bytes(st())                                   # None = the all-zero default
        nat.set_input_transform(o, input_transform_of(tl_val_pipeline))
        assert o.in_swap_rb == 1 and F32(o.in_mean[0]) == F32(0.485) * F32(255) and o.in_scale[2] > 0


def _stem_op(transform=None, **over):
    o = nat.Op()
    o.kind, o.dtype = nat.OP_STEM0, nat.DTYPE_BF16
    o.N, o.H, o.W, o.Cin, o.Ho, o.Wo, o.Cout = 1, 32, 32, 3, 16, 16, 64
    o.ksize, o.stride, o.relu = 3, 2, 1
    o.in_off, o.out_off, o.res_off, o.stats_off, o.ds_out_off = -1, 4096, -1, -1, -1
    o.weight = 256
    nat.set_input_transform(o, transform)
    for k, v in over.items():
        if isinstance(v, tuple):
            getattr(o, k)[:] = v
        else:
            setattr(o, k, v)
    return o


def _plan_rc(o):
    """Plans the op, enqueues nothing: without an input pointer lfd_run_op stops right after planning (LFD_ERR_INVALID 'needs the external
    input pointer'); without a device it stops before it (LFD_ERR_CUDA).  -> (rc, message)"""
    ws = (C.c_uint8 * 16)()
    rc = nat.lib().lfd_run_op(C.byref(o), None, nat.INPUT_U8_NHWC, C.addressof(ws), None, None, 0, 0, nat.CONV_UMMA, None)
    return rc, nat.lib().lfd_last_error().decode()


@pytest.mark.skipif(not torch.cuda.is_available(), reason='lfd_run_op plans ops only when a device is present')
def test_partly_set_transforms_are_invalid_and_zero_is_the_simple_constants():
    inv = float(F32(1) / F32(127.5))
    for o in (_stem_op(), _stem_op(InputTransform(False, (127.5,) * 3, (inv,) * 3)), _stem_op(input_transform_of(tl_val_pipeline))):
        rc, msg = _plan_rc(o)
        assert rc == 1 and 'external input pointer' in msg, msg         # planned, then stopped for want of an image
    bad = [dict(in_mean=(127.5, 127.5, 127.5)),                            # means without scales
           dict(in_swap_rb=1),                                             # a swap alone
           dict(in_mean=(1.0, 1.0, 1.0), in_scale=(1.0, 0.0, 1.0)),        # one zero scale
           dict(in_scale=(1.0, float('inf'), 1.0)), dict(in_scale=(1.0, 1.0, 1.0), in_mean=(float('nan'), 0.0, 0.0)),
           dict(in_swap_rb=2, in_scale=(1.0, 1.0, 1.0))]
    for over in bad:
        rc, msg = _plan_rc(_stem_op(**over))
        assert rc == 1 and 'input transform' in msg, (over, msg)


def _models():
    yield 'TL_L', synth_model('TL_L')[0], None
    yield 'TL_S', tl_s.synth_model()[0], None
    yield 'WIDERFACE_S', synth_model('WIDERFACE_S')[0], True


@pytest.mark.parametrize('pipeline', [tl_val_pipeline, typical_coco_val_pipeline], ids=['tl', 'coco'])
def test_the_transform_reaches_the_stem_op_and_only_it(pipeline):
    t = input_transform_of(pipeline)
    for name, model, fuse in _models():
        base = InferencePlan(model, 2, 256, 320, 'cpu', create_native=False, fuse_stem=fuse)
        plan = InferencePlan(model, 2, 256, 320, 'cpu', create_native=False, fuse_stem=fuse, input_transform=t)
        assert plan._ops[0]['kind'] == (nat.OP_STEM4 if fuse else nat.OP_STEM0), name
        assert len(plan._op_array) == len(base._op_array)
        for i, (a, b) in enumerate(zip(plan._op_array, base._op_array)):
            got = (a.in_swap_rb, tuple(a.in_mean), tuple(a.in_scale))
            assert got == ((int(t.swap_rb), _f32(*t.mean), _f32(*t.scale)) if i == 0 else (0, (0.0,) * 3, (0.0,) * 3)), (name, i)
            assert (b.in_swap_rb, tuple(b.in_mean), tuple(b.in_scale)) == (0, (0.0,) * 3, (0.0,) * 3)
            assert (a.kind, a.H, a.W, a.Cout, a.out_off) == (b.kind, b.H, b.W, b.Cout, b.out_off)


def test_the_transform_is_part_of_the_plan_cache_keys(monkeypatch):
    import lfd.model.lfd as lfd_module
    import lfd._train as train_module
    built = []

    class FakePlan(object):
        def __init__(self, model, *a, **kw):
            self.input_transform = kw.get('input_transform', getattr(model, 'input_transform', None))
            built.append(self.input_transform)

    monkeypatch.setattr(lfd_module, 'InferencePlan', FakePlan)
    monkeypatch.setattr(train_module, 'TrainPlan', FakePlan)
    monkeypatch.setattr(train_module, 'flat_parameters', lambda model: None)
    model = synth_model('TL_L')[0]
    for plan_for in (lambda: model.inference_plan(2, 64, 64, 'cpu'), lambda: model.train_plan_for(2, 64, 64, 'cpu')):
        del built[:]
        model.set_input_transform(None)
        a = plan_for()
        model.set_input_transform(tl_val_pipeline)
        b = plan_for()
        model.set_input_transform(typical_coco_val_pipeline)
        c = plan_for()
        model.set_input_transform(tl_val_pipeline)
        assert plan_for() is b and a is not b and b is not c
        model.set_input_transform(None)
        assert plan_for() is a
        assert built == [None, input_transform_of(tl_val_pipeline), input_transform_of(typical_coco_val_pipeline)]


def test_training_plan_and_frozen_prefix_carry_the_transform():
    from lfd._train import TrainPlan
    t = input_transform_of(tl_val_pipeline)
    want = (1, _f32(*t.mean), _f32(*t.scale))

    def fields(o):
        return o.in_swap_rb, tuple(o.in_mean), tuple(o.in_scale)

    model = synth_model('TL_L')[0]
    model.train()
    model.set_input_transform(tl_val_pipeline)
    plan = TrainPlan(model, 2, 128, 160, 'cpu', create_native=False)
    seen = []
    for ops, arr in ((plan.fwd_ops, plan._fwd_arr), (plan.bwd_ops, plan._bwd_arr)):
        for op, o in zip(ops, arr):
            if op['kind'] in (nat.TOP_STEM0, nat.TOP_WGRAD_STEM):
                seen.append(op['kind'])
                assert fields(o) == want
            else:
                assert fields(o) == (0, (0.0,) * 3, (0.0,) * 3)
    assert seen == [nat.TOP_STEM0, nat.TOP_WGRAD_STEM]
    # fine-tuning: the frozen prefix's stem is an inference op inside the training plan
    from test_finetune_plan import finetune_model
    frozen = finetune_model('WIDERFACE_L', 1)
    frozen.set_input_transform(tl_val_pipeline)
    plan = TrainPlan(frozen, 2, 128, 160, 'cpu', create_native=False)
    assert plan._prefix is not None
    ops = plan._prefix['arr']
    assert ops[0].kind in (nat.OP_STEM0, nat.OP_STEM4) and fields(ops[0]) == want
    assert all(fields(o) == (0, (0.0,) * 3, (0.0,) * 3) for o in list(ops)[1:])
    assert all(op['kind'] not in (nat.TOP_STEM0, nat.TOP_WGRAD_STEM) for op in plan.fwd_ops + plan.bwd_ops)


def test_loader_exposes_the_transform_only_when_asked():
    from lfd.data_pipeline.data_loader import DataLoader

    class Sampler(object):
        def __len__(self):
            return 0

        def get_batch_size(self):
            return 2

    class Region(object):
        def draw(self, *a, **kw):
            raise AssertionError

    pipe = Compose([HorizontalFlip(p=0.5), BGR2RGB(), standard_normalize], bbox_params=bbox_param)
    assert DataLoader(None, Sampler(), Region(), pipe).input_transform is None
    assert DataLoader(None, Sampler(), Region(), pipe, model_normalizes=True).input_transform == input_transform_of(tl_val_pipeline)
    with pytest.raises(ValueError):
        DataLoader(None, Sampler(), Region(), opaque(pipe), model_normalizes=True)

