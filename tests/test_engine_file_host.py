# -*- coding: utf-8 -*-
"""Model files on the host: export every shipped config without a device (create_native=False), read the file back through the C ABI
(lfd_engine_open / lfd_engine_info / lfd_engine_op) and compare it with the plan; the export is deterministic; and lfd_engine_open
refuses corrupted files with the documented code and a message that names the field."""
import ctypes as C
import struct
import zlib

import pytest
import torch

from helpers import model_of
from lfd import _native as nat
from lfd._engine import MODEL_FORMAT_VERSION
from lfd.deployment import export_model
from test_input_transform_host import tl_val_pipeline

LFD_ERR_INVALID, LFD_ERR_UNSUPPORTED = 1, 3
CONFIGS = ['WIDERFACE_XS', 'WIDERFACE_S', 'WIDERFACE_M', 'WIDERFACE_L', 'TT100K_S', 'TT100K_L', 'TL_L', 'TL_S']
PTR_FIELDS = [n for n, t in nat.Op._fields_ if t is C.c_void_p]
HEADER, PLAN = 48, 120


def export(tmp_path, name, N=2, H=200, W=264, tag='a', **kw):
    path = str(tmp_path / ('%s_%s.lfd' % (name, tag)))
    pipeline = tl_val_pipeline if name.startswith('TL') else None
    plan, post = export_model(model_of(name), path, N, H, W, input_pipeline=pipeline, create_native=False, **kw)
    return plan, post, open(path, 'rb').read()


def open_engine(data):
    """-> (return code, engine handle or None, lfd_last_error())"""
    lib = nat.lib()
    e = C.c_void_p()
    rc = lib.lfd_engine_open(data, len(data), C.byref(e))
    msg = lib.lfd_last_error().decode()
    return rc, (e if rc == 0 else None), msg


def blob_of(plan, ptr):
    """A pointer of the plan's op array -> (blob, byte offset) in the two staging buffers, or None for NULL."""
    if not ptr:
        return None
    for blob, t in enumerate((plan.params_f32, plan.params_bf16)):
        base = t.data_ptr()
        if base <= ptr < base + t.numel() * t.element_size():
            return blob, ptr - base
    raise AssertionError('pointer outside the staging buffers')


@pytest.mark.parametrize('name', CONFIGS)
def test_round_trip(tmp_path, name):
    plan, post, data = export(tmp_path, name)
    rc, e, msg = open_engine(data)
    assert rc == 0, msg
    lib = nat.lib()
    try:
        d = nat.EngineDesc()
        nat.check(lib.lfd_engine_info(e, C.byref(d)))
        assert (d.N, d.H, d.W, d.P, d.cls_channels, d.n_ops) == (2, 200, 264, plan.P, plan.cls_channels, len(plan._ops))
        assert (d.num_classes, d.dtype, d.cap, d.soft_nms) == (post.cfg.C, nat.DTYPE_BF16, post.cfg.cap, 0)
        assert d.workspace_bytes >= plan.workspace_bytes + 4 * plan.N * plan.P * (plan.cls_channels + 4)
        assert d.weights_bytes >= plan.params_f32.numel() * 4 + plan.params_bf16.numel() * 2
        assert d.post_workspace_bytes >= lib.lfd_postprocess_workspace_bytes(C.byref(post.cfg))
        assert lib.lfd_engine_num_launches(e) == 0          # not bound
        writer = {}
        for i, want in enumerate(plan._op_array):
            got, src, level = nat.Op(), C.c_int32(), C.c_int32()
            nat.check(lib.lfd_engine_op(e, i, C.byref(got), C.byref(src), C.byref(level)))
            for f, t in nat.Op._fields_:
                g, w = getattr(got, f), getattr(want, f)
                if t is C.c_void_p:
                    v = g or 0
                    assert (None if v == 0 else ((v >> 56) - 1, v & ((1 << 56) - 1))) == blob_of(plan, w), (name, i, f)
                elif f in ('in_mean', 'in_scale'):
                    assert list(g) == list(w), (name, i, f)
                else:
                    assert g == w, (name, i, f, g, w)
            # the producer of the op's input and the head level
            if i == 0:
                assert src.value == -1
            else:
                assert 0 <= src.value < i and got.in_off in (writer[src.value]), (name, i, src.value)
            assert level.value == (plan._ops[i]['level'] if got.kind == nat.OP_HEAD_FINAL else -1)
            writer[i] = (got.out_off, got.ds_out_off)
        assert lib.lfd_engine_op(e, len(plan._ops), C.byref(nat.Op()), None, None) == LFD_ERR_INVALID
    finally:
        lib.lfd_engine_close(e)


def test_input_transform_and_soft_nms_are_in_the_file(tmp_path):
    model = model_of('TL_L')
    old = dict(model._nms_cfg)
    model._nms_cfg = dict(type='soft_nms', iou_thr=0.35, method='gaussian', sigma=0.7, min_score=0.01)
    try:
        plan, post, data = export(tmp_path, 'TL_L', classification_threshold=0.25, class_agnostic=True)
    finally:
        model._nms_cfg = old
    p = HEADER
    swap, = struct.unpack_from('<i', data, p + 56)
    mean, scale = struct.unpack_from('<3f', data, p + 60), struct.unpack_from('<3f', data, p + 72)
    soft = struct.unpack_from('<ii2f', data, p + 84)
    xf = plan.input_transform
    assert swap == 1 and list(mean) == list(torch.tensor(xf.mean, dtype=torch.float32).tolist())
    assert list(scale) == list(torch.tensor(xf.scale, dtype=torch.float32).tolist())
    assert soft[:2] == (1, 2) and soft[2] == pytest.approx(0.7) and soft[3] == pytest.approx(0.01)
    cfg = nat.PostCfg.from_buffer_copy(data[p + PLAN:p + PLAN + C.sizeof(nat.PostCfg)])
    assert cfg.class_agnostic == 1 and cfg.score_thr == pytest.approx(0.25) and cfg.iou_thr == pytest.approx(0.35)
    rc, e, msg = open_engine(data)
    assert rc == 0, msg
    d = nat.EngineDesc()
    nat.check(nat.lib().lfd_engine_info(e, C.byref(d)))
    assert d.soft_nms == 1
    nat.lib().lfd_engine_close(e)


def test_two_exports_are_byte_identical(tmp_path):
    for name in ('WIDERFACE_S', 'TL_S'):
        a = export(tmp_path, name, tag='a')[2]
        b = export(tmp_path, name, tag='b')[2]
        assert a == b, name


def test_export_refuses_a_pipeline_the_kernels_cannot_run(tmp_path):
    from lfd.data_pipeline.augmentation import Compose, HorizontalFlip
    with pytest.raises(ValueError):
        export_model(model_of('TL_L'), str(tmp_path / 'x.lfd'), 1, 64, 64, input_pipeline=Compose([HorizontalFlip(p=0.5)]), create_native=False)


# ------------------------------------------------------------------------------------------------------------------ rejection
def resign(b):
    """The file with its header's payload size and CRC-32 recomputed, so that a corruption reaches the field checks."""
    b = bytearray(b)
    payload = bytes(b[HEADER:])
    struct.pack_into('<QI', b, 32, len(payload), zlib.crc32(payload))
    return bytes(b)


def sections(data):
    """-> the byte offsets where the file's sections end."""
    n_ops, = struct.unpack_from('<i', data, HEADER + 28)
    b0, b1 = struct.unpack_from('<2q', data, HEADER + 104)
    ends = [HEADER, HEADER + PLAN, HEADER + PLAN + C.sizeof(nat.PostCfg)]
    ends.append(ends[-1] + n_ops * C.sizeof(nat.Op))
    ends.append(ends[-1] + n_ops * 8)
    ends.append(ends[-1] + b0)
    ends.append(ends[-1] + b1)
    assert ends[-1] == len(data)
    return ends


def op_at(data, i):
    return HEADER + PLAN + C.sizeof(nat.PostCfg) + i * C.sizeof(nat.Op)


def refused(data, code, field):
    rc, e, msg = open_engine(data)
    if e is not None:
        nat.lib().lfd_engine_close(e)
    assert rc == code and field in msg, (rc, msg)
    return msg


@pytest.fixture(scope='module')
def model_file(tmp_path_factory):
    plan, _, data = export(tmp_path_factory.mktemp('model'), 'WIDERFACE_S', N=1, H=128, W=160)
    assert open_engine(data)[0] == 0
    return plan, data


def test_truncated_files(model_file):
    _, data = model_file
    for n in [0, 7, 47] + sections(data)[:-1] + [len(data) - 1]:
        refused(data[:n], LFD_ERR_INVALID, 'header' if n < HEADER else 'payload_bytes')
    refused(data + b'\0', LFD_ERR_INVALID, 'payload_bytes')
    # a header that agrees with a truncated payload still needs every section
    for n in sections(data)[:-1]:
        refused(resign(data[:n]), LFD_ERR_INVALID, 'payload_bytes' if n < sections(data)[2] else 'payload_bytes =')


def test_header_fields(model_file):
    _, data = model_file

    def patched(off, fmt, value):
        b = bytearray(data)
        struct.pack_into(fmt, b, off, value)
        return bytes(b)
    refused(patched(0, '<8s', b'LFDMODEM'), LFD_ERR_INVALID, 'magic')
    refused(patched(8, '<I', MODEL_FORMAT_VERSION + 1), LFD_ERR_UNSUPPORTED, 'format version')
    refused(patched(12, '<I', nat.ABI_VERSION - 1), LFD_ERR_UNSUPPORTED, 'abi version')
    refused(patched(16, '<8s', b'sm_100a'), LFD_ERR_UNSUPPORTED, 'target')
    refused(patched(24, '<I', C.sizeof(nat.Op) - 8), LFD_ERR_INVALID, 'lfd_op struct bytes')
    refused(patched(28, '<I', C.sizeof(nat.PostCfg) + 4), LFD_ERR_INVALID, 'lfd_post_cfg struct bytes')
    refused(patched(44, '<I', 1), LFD_ERR_INVALID, 'reserved')


def test_checksum(model_file):
    _, data = model_file
    for at in (len(data) - 3, sections(data)[-2] + 5, HEADER + 1):       # a 16-bit weight, an fp32 parameter, the plan
        b = bytearray(data)
        b[at] ^= 0x10
        refused(bytes(b), LFD_ERR_INVALID, 'checksum')


def test_field_checks(model_file):
    plan, data = model_file
    n_ops = len(plan._ops)

    def patched(off, fmt, value):
        b = bytearray(data)
        struct.pack_into(fmt, b, off, value)
        return resign(b)
    conv = next(i for i, op in enumerate(plan._ops) if op['kind'] == nat.OP_CONV)
    head = next(i for i, op in enumerate(plan._ops) if op['kind'] == nat.OP_HEAD_FINAL)
    for kind in (5, 9, -1, 1 << 20):
        refused(patched(op_at(data, conv) + nat.Op.kind.offset, '<i', kind), LFD_ERR_INVALID, 'kind %d' % kind)
    ws = plan.workspace_bytes
    for field in ('out_off', 'in_off'):
        for off in (ws, ws - 256, 1 << 50, -2):
            refused(patched(op_at(data, conv) + getattr(nat.Op, field).offset, '<q', off), LFD_ERR_INVALID, field)
    refused(patched(op_at(data, head) + nat.Op.stats_off.offset, '<q', ws), LFD_ERR_INVALID, 'stats_off')
    # pointers: past the blob, in the other blob, an unknown blob
    b16, f32 = plan.params_bf16.numel() * 2, plan.params_f32.numel() * 4
    for field, value in (('weight', (2 << 56) | b16), ('weight', (2 << 56) | (b16 - 16)), ('weight', 1 << 56), ('weight', 3 << 56),
                         ('shift', (1 << 56) | f32), ('tail_scale', 1 << 56)):
        refused(patched(op_at(data, conv) + getattr(nat.Op, field).offset, '<Q', value), LFD_ERR_INVALID, field)
    refused(patched(op_at(data, head) + nat.Op.weight.offset, '<Q', (1 << 56) | (f32 - 4)), LFD_ERR_INVALID, 'weight')
    # the op count and the other plan fields
    for n in (0, -1, -(1 << 31), 1 << 30, 4097, n_ops + 1, n_ops - 1):
        refused(patched(HEADER + 28, '<i', n), LFD_ERR_INVALID, 'n_ops' if not 1 <= n <= 4096 else 'payload_bytes')
    refused(patched(HEADER + 0, '<i', 0), LFD_ERR_INVALID, 'capacity')
    refused(patched(HEADER + 4, '<i', 1 << 20), LFD_ERR_INVALID, 'capacity')
    refused(patched(HEADER + 48, '<q', 1 << 62), LFD_ERR_INVALID, 'workspace_bytes')
    refused(patched(HEADER + 48, '<q', ws - 256), LFD_ERR_INVALID, 'workspace')
    refused(patched(HEADER + 20, '<i', 7), LFD_ERR_INVALID, 'dtype')
    refused(patched(HEADER + 24, '<i', nat.CONV_SIMT), LFD_ERR_UNSUPPORTED, 'conv_impl')
    refused(patched(HEADER + 84, '<i', 2), LFD_ERR_INVALID, 'nms_type')
    refused(patched(HEADER + 56, '<i', 3), LFD_ERR_INVALID, 'input transform')
    refused(patched(HEADER + PLAN + nat.PostCfg.cap.offset, '<i', 0), LFD_ERR_INVALID, 'cap')
    refused(patched(HEADER + PLAN + nat.PostCfg.P.offset, '<i', plan.P + 1), LFD_ERR_INVALID, 'post-process N / P')
    # the producer / level table
    aux = op_at(data, n_ops)
    refused(patched(aux + 8 * conv, '<i', conv), LFD_ERR_INVALID, 'src_op')
    refused(patched(aux + 8 * conv, '<i', -5), LFD_ERR_INVALID, 'src_op')
    refused(patched(aux + 8 * head + 4, '<i', 9), LFD_ERR_INVALID, 'level')
    refused(patched(aux + 4, '<i', 0), LFD_ERR_INVALID, 'level')
    # geometry the plan checks as well
    refused(patched(op_at(data, conv) + nat.Op.Ho.offset, '<i', 1 << 20), LFD_ERR_INVALID, 'Ho')
    # the image op reads frames of the capacity lfd_engine_info reports, which the caller sizes its input by
    for field, value in (('H', 129), ('W', 161), ('H', 127)):
        refused(patched(op_at(data, 0) + getattr(nat.Op, field).offset, '<i', value), LFD_ERR_INVALID, 'capacity')
    refused(patched(HEADER + 4, '<i', 130), LFD_ERR_INVALID, 'capacity')
    # what lfd_plan_create or a launch would refuse later
    refused(patched(op_at(data, head) + nat.Op.n_reg.offset, '<i', 2), LFD_ERR_INVALID, 'n_reg')
    for field, value in (('stride', 0), ('stride', 3), ('ksize', 5)):
        refused(patched(op_at(data, conv) + getattr(nat.Op, field).offset, '<i', value), LFD_ERR_INVALID, field)
    refused(patched(op_at(data, conv) + nat.Op.cc.offset, '<i', plan._op_array[conv].cc // 2), LFD_ERR_INVALID, 'cc')
    # an op reads an output of its producer, with the producer's channel count
    refused(patched(op_at(data, conv) + nat.Op.in_off.offset, '<q', plan._op_array[conv].out_off), LFD_ERR_INVALID, 'in_off')
    narrow = next(i for i, o in enumerate(plan._op_array) if o.kind == nat.OP_CONV and o.Cin >= 32 and not o.ds_cout and not o.tail_cout)
    o = plan._op_array[narrow]
    cc = nat.conv_query(o.N, o.H, o.W, o.Cin // 2, o.Ho, o.Wo, o.Cout, o.ksize, o.stride)['cc']
    b = bytearray(data)
    struct.pack_into('<i', b, op_at(data, narrow) + nat.Op.Cin.offset, o.Cin // 2)
    struct.pack_into('<i', b, op_at(data, narrow) + nat.Op.cc.offset, cc)
    refused(resign(b), LFD_ERR_INVALID, 'Cin = %d' % (o.Cin // 2))
    # the input transform that runs (op 0's) is the plan's; no other op carries one
    refused(patched(op_at(data, 0) + nat.Op.in_swap_rb.offset, '<i', 1), LFD_ERR_INVALID, 'input transform')
    refused(patched(op_at(data, conv) + nat.Op.in_scale.offset, '<f', 1.0), LFD_ERR_INVALID, 'input transform')
    refused(patched(HEADER + 100, '<i', 1), LFD_ERR_INVALID, 'reserved')


def test_fused_stem_at_another_size_than_the_capacity(tmp_path):
    """A fused stem's output size does not change between 125 x 157 and 128 x 160: the image op's own size is checked against the
    capacity, or the kernel would read a 160-pixel pitch in a buffer of 157-pixel rows."""
    from lfd._engine import InferencePlan, PostPlan
    model = model_of('WIDERFACE_S')
    plan = InferencePlan(model, 1, 125, 157, torch.device('cpu'), create_native=False, fuse_stem=True)
    assert plan._ops[0]['kind'] == nat.OP_STEM4
    post = PostPlan(model._post_cfg(1, plan.level_sizes, 0.3, 0.4, False), torch.device('cpu'))
    data = plan.model_file_bytes(post)
    assert open_engine(data)[0] == 0
    b = bytearray(data)
    struct.pack_into('<ii', b, op_at(data, 0) + nat.Op.H.offset, 128, 160)
    refused(resign(b), LFD_ERR_INVALID, 'capacity')
