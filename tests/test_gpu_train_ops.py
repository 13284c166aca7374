# -*- coding: utf-8 -*-
"""Per-kernel parity of the native training ops against torch autograd (fp32, CPU) on the SAME 16-bit operands: parameter
staging, BatchNorm batch statistics / apply, BatchNorm / GroupNorm backward, head-final backward, data gradients (the forward
wgmma kernel on transposed / flipped weights, zero-inserted for stride 2), weight gradients (wgmma MN-major kernel, SIMT
cross-check, stem), clip + SGD.  Reference semantics: torch.nn modules as the reference uses them (lfd_resnet.py:10-18,96-154,
lfd_head.py:85-185, optimizer_hook.py:21-36)."""
import pytest
import torch
import torch.nn.functional as F

from lfd import _native as nat
from lfd._engine import pack_conv_weight, pack_stem_weight
from gpu_train_ops import Workspace, make_top, run_top, desc_table, bf16r

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def conv_out(size, k, s):
    return (size + 2 * (k // 2) - k) // s + 1


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))


# ------------------------------------------------------------------------------------------------ staging
@pytest.mark.parametrize('cout,cin,k', [(64, 64, 3), (128, 64, 1), (64, 128, 3), (32, 32, 1)])
def test_pack_conv_forward_and_dgrad(cout, cin, k):
    torch.manual_seed(1)
    w = torch.randn(cout, cin, k, k)
    cc_f = 32 if cin % 64 else 64
    cc_d = 32 if cout % 64 else 64
    wd = w.to(DEV)
    out_f = torch.zeros(w.numel(), dtype=torch.bfloat16, device=DEV)
    out_d = torch.zeros(w.numel(), dtype=torch.bfloat16, device=DEV)
    d1 = nat.PackDesc(kind=nat.PACK_CONV_FWD, Cout=cout, Cin=cin, k=k, cc=cc_f, n=w.numel(), src=wd.data_ptr(), dst=out_f.data_ptr())
    d2 = nat.PackDesc(kind=nat.PACK_CONV_DGRAD, Cout=cout, Cin=cin, k=k, cc=cc_d, n=w.numel(), src=wd.data_ptr(), dst=out_d.data_ptr())
    table = desc_table([d1, d2], DEV)
    ws = Workspace(DEV).finalize()
    run_top(make_top(nat.TOP_PACK, n_desc=2, max_n=w.numel(), ptr={0: table.data_ptr()}), ws)
    assert torch.equal(out_f.cpu().view(-1), pack_conv_weight(w, cc_f).view(-1))
    wt = w.permute(1, 0, 2, 3).flip(2, 3).contiguous()          # the transposed conv's OIHW weights
    assert torch.equal(out_d.cpu().view(-1), pack_conv_weight(wt, cc_d).view(-1))


def test_pack_stem_round_and_scale_shift():
    torch.manual_seed(2)
    w = torch.randn(64, 3, 3, 3).to(DEV)
    hw = torch.randn(5, 128).to(DEV)
    bias = torch.randn(4).to(DEV)
    scale = torch.tensor(1.7).to(DEV)
    o_stem = torch.zeros(3 * 2 * 64 * 8, dtype=torch.bfloat16, device=DEV)
    o_hw = torch.zeros(5 * 128, device=DEV)
    o_s, o_sh, o_b = torch.zeros(4, device=DEV), torch.zeros(4, device=DEV), torch.zeros(4, device=DEV)
    ds = [nat.PackDesc(kind=nat.PACK_STEM, Cout=64, Cin=3, k=3, cc=0, n=o_stem.numel(), src=w.data_ptr(), dst=o_stem.data_ptr()),
          nat.PackDesc(kind=nat.PACK_ROUND_F32, n=o_hw.numel(), src=hw.data_ptr(), dst=o_hw.data_ptr()),
          nat.PackDesc(kind=nat.PACK_SCALE_SHIFT, n=4, src=bias.data_ptr(), src2=scale.data_ptr(), dst=o_s.data_ptr(), dst2=o_sh.data_ptr(), dst3=o_b.data_ptr())]
    table = desc_table(ds, DEV)
    ws = Workspace(DEV).finalize()
    run_top(make_top(nat.TOP_PACK, n_desc=3, max_n=o_stem.numel(), ptr={0: table.data_ptr()}), ws)
    assert torch.equal(o_stem.cpu().view(-1), pack_stem_weight(w.cpu()).view(-1))
    assert torch.equal(o_hw.cpu(), bf16r(hw.cpu()).view(-1))
    assert torch.allclose(o_s.cpu(), torch.full((4,), 1.7)) and torch.allclose(o_sh.cpu(), bias.cpu() * 1.7) and torch.equal(o_b.cpu(), bias.cpu())


def test_unpack_conv_and_add():
    torch.manual_seed(3)
    stage = torch.randn(9, 32, 64).to(DEV)        # [tap][ci][co]
    grad = torch.randn(64, 32, 3, 3).to(DEV)
    g0 = grad.clone()
    a, b = torch.randn(100).to(DEV), torch.randn(100).to(DEV)
    b0 = b.clone()
    ds = [nat.UnpackDesc(kind=nat.UNPACK_CONV, Cout=64, Cin=32, kk=9, n=grad.numel(), src=stage.data_ptr(), dst=grad.data_ptr()),
          nat.UnpackDesc(kind=nat.UNPACK_ADD, n=100, src=a.data_ptr(), dst=b.data_ptr())]
    table = desc_table(ds, DEV)
    ws = Workspace(DEV).finalize()
    run_top(make_top(nat.TOP_UNPACK, n_desc=2, max_n=grad.numel(), ptr={0: table.data_ptr()}), ws)
    want = g0 + stage.permute(2, 1, 0).reshape(64, 32, 3, 3)
    assert torch.allclose(grad, want) and torch.allclose(b, a + b0)


# ------------------------------------------------------------------------------------------------ BatchNorm
@pytest.mark.parametrize('C,res,relu', [(64, True, True), (128, False, True), (32, False, False)])
def test_bn_train_forward_and_backward(C, res, relu):
    torch.manual_seed(4)
    N, H, W = 3, 13, 11
    z = bf16r(torch.randn(N, H, W, C) * 2 + 0.5)
    r = bf16r(torch.randn(N, H, W, C)) if res else None
    gamma, beta = torch.rand(C) + 0.5, torch.randn(C) * 0.2
    rm, rv = torch.randn(C) * 0.1, torch.rand(C) + 0.5
    dy = bf16r(torch.randn(N, H, W, C))
    ws = Workspace(DEV)
    ws.add('z', z.to(torch.bfloat16))
    ws.add('y', shape=(N, H, W, C), dtype=torch.bfloat16)
    if res:
        ws.add('res', r.to(torch.bfloat16))
    ws.add('sums', shape=(C, 2), dtype=torch.float64)
    ws.add('bsums', shape=(C, 2), dtype=torch.float64)
    ws.add('dy', dy.to(torch.bfloat16))
    ws.add('dz', shape=(N, H, W, C), dtype=torch.bfloat16)
    ws.add('dres', shape=(N, H, W, C), dtype=torch.bfloat16)
    ws.add('dzu', shape=(N, 2 * H, 2 * W - 1, C), dtype=torch.bfloat16)
    ws.finalize()
    g_d, b_d, rm_d, rv_d = gamma.to(DEV), beta.to(DEV), rm.to(DEV), rv.to(DEV)
    dg_d, db_d = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    geo = dict(N=N, H=H, W=W, Cout=C, eps=1e-5)
    run_top(make_top(nat.TOP_BN_STATS, off={0: ws.off('z'), 3: ws.off('sums')}, **geo), ws)
    run_top(make_top(nat.TOP_BN_APPLY, relu=int(relu), momentum=0.1, off={0: ws.off('z'), 1: ws.off('y'), 2: ws.off('res') if res else -1, 3: ws.off('sums')},
                     ptr={0: g_d.data_ptr(), 1: b_d.data_ptr(), 2: rm_d.data_ptr(), 3: rv_d.data_ptr()}, **geo), ws)
    # torch reference (fp32) on the same stored z
    zt = z.permute(0, 3, 1, 2).clone().requires_grad_(True)
    gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rt = r.permute(0, 3, 1, 2).clone().requires_grad_(True) if res else None
    rm_t, rv_t = rm.clone(), rv.clone()
    yt = F.batch_norm(zt, rm_t, rv_t, gt, bt, training=True, momentum=0.1, eps=1e-5)
    if res:
        yt = yt + rt
    if relu:
        yt = F.relu(yt)
    y = ws.get('y').float().cpu()
    want = yt.detach().permute(0, 2, 3, 1)
    assert float((y - want).abs().max()) <= 2.0 ** -7 * float(want.abs().max()) + 1e-6
    assert torch.allclose(rm_d.cpu(), rm_t, atol=1e-5) and torch.allclose(rv_d.cpu(), rv_t, atol=1e-5, rtol=1e-5)
    # backward: the mask comes from the STORED y, so feed torch the same decision by differentiating at the stored output
    yt.backward(dy.permute(0, 3, 1, 2))
    offs = {0: ws.off('dy'), 1: ws.off('y') if relu else -1, 2: ws.off('z'), 3: ws.off('sums'), 4: ws.off('bsums')}
    run_top(make_top(nat.TOP_NORM_BWD_REDUCE, relu=int(relu), off=offs, ptr={0: g_d.data_ptr(), 1: b_d.data_ptr()}, **geo), ws)
    offs.update({5: ws.off('dz'), 6: ws.off('dzu'), 7: ws.off('dres') if res else -1})
    run_top(make_top(nat.TOP_NORM_BWD_APPLY, relu=int(relu), upH=2 * H, upW=2 * W - 1, off=offs,
                     ptr={0: g_d.data_ptr(), 1: b_d.data_ptr(), 2: dg_d.data_ptr(), 3: db_d.data_ptr()}, **geo), ws)
    dz = ws.get('dz').float().cpu()
    want_dz = zt.grad.permute(0, 2, 3, 1)
    assert rel(dz, want_dz) < 1.2e-2, rel(dz, want_dz)          # bf16 storage of dz: 2^-8 relative per element
    assert rel(dg_d, gt.grad) < 2e-3 and rel(db_d, bt.grad) < 2e-3
    if res:
        assert rel(ws.get('dres').float(), rt.grad.permute(0, 2, 3, 1)) < 1e-6
    dzu = ws.get('dzu').float().cpu()
    assert torch.equal(dzu[:, ::2, ::2, :], dz)
    mask = torch.ones_like(dzu, dtype=torch.bool)
    mask[:, ::2, ::2, :] = False
    assert float(dzu[mask].abs().max()) == 0.0


def test_gn_backward():
    torch.manual_seed(5)
    N, H, W, C, G = 2, 9, 7, 128, 16
    raw = bf16r(torch.randn(N, H, W, C) * 1.5)
    gamma, beta = torch.rand(C) + 0.5, torch.randn(C) * 0.3
    dact = bf16r(torch.randn(N, H, W, C))
    x = raw.reshape(N, H * W, G, 8).double()
    stats = torch.stack([x.sum((1, 3)), (x * x).sum((1, 3))], -1)      # [N][G][2]
    ws = Workspace(DEV)
    ws.add('raw', raw.to(torch.bfloat16))
    ws.add('stats', stats)
    ws.add('bsums', shape=(C * 2 + N * G * 2,), dtype=torch.float64)
    ws.add('dact', dact.to(torch.bfloat16))
    ws.add('draw', shape=(N, H, W, C), dtype=torch.bfloat16)
    ws.finalize()
    g_d, b_d = gamma.to(DEV), beta.to(DEV)
    dg_d, db_d = torch.zeros(C, device=DEV), torch.zeros(C, device=DEV)
    geo = dict(N=N, H=H, W=W, Cout=C, groups=G, relu=1, eps=1e-5)
    offs = {0: ws.off('dact'), 2: ws.off('raw'), 3: ws.off('stats'), 4: ws.off('bsums')}
    run_top(make_top(nat.TOP_NORM_BWD_REDUCE, off=offs, ptr={0: g_d.data_ptr(), 1: b_d.data_ptr()}, **geo), ws)
    offs[5] = ws.off('draw')
    run_top(make_top(nat.TOP_NORM_BWD_APPLY, off=offs, ptr={0: g_d.data_ptr(), 1: b_d.data_ptr(), 2: dg_d.data_ptr(), 3: db_d.data_ptr()}, **geo), ws)
    rt = raw.permute(0, 3, 1, 2).clone().requires_grad_(True)
    gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    F.relu(F.group_norm(rt, G, gt, bt, 1e-5)).backward(dact.permute(0, 3, 1, 2))
    got = ws.get('draw').float()
    assert rel(got, rt.grad.permute(0, 2, 3, 1)) < 1.2e-2
    assert rel(dg_d, gt.grad) < 2e-3 and rel(db_d, bt.grad) < 2e-3


# ------------------------------------------------------------------------------------------------ head final
@pytest.mark.parametrize('n_cls,n_reg', [(1, 4), (46, 0), (0, 4)])
def test_head_final_forward_and_backward(n_cls, n_reg):
    torch.manual_seed(6)
    N, H, W, C, G = 2, 11, 13, 128, 16
    HW, P, point_off = H * W, H * W + 37, 20
    no = n_cls + n_reg
    raw = bf16r(torch.randn(N, HW, C))
    gamma, beta = torch.rand(C) + 0.5, torch.randn(C) * 0.3
    wf = bf16r(torch.randn(no, C) * 0.1)
    bias = torch.randn(no) * 0.1
    scale = torch.cat([torch.ones(n_cls), torch.full((n_reg,), 1.3)])
    x = raw.reshape(N, HW, G, 8).double()
    stats = torch.stack([x.sum((1, 3)), (x * x).sum((1, 3))], -1)
    gcls = torch.randn(N, P, max(n_cls, 1)) * (n_cls > 0)
    greg = torch.randn(N, P, 4) * (n_reg > 0)
    ws = Workspace(DEV)
    ws.add('raw', raw.to(torch.bfloat16))
    ws.add('stats', stats)
    ws.add('stage', torch.cat([wf.reshape(-1), scale, bias * scale, bias]))
    ws.add('dstage', shape=(no * C + no,), dtype=torch.float32)
    ws.add('dscale', shape=(1,), dtype=torch.float32)
    ws.add('dact', shape=(N, HW, C), dtype=torch.bfloat16)
    ws.finalize()
    g_d, b_d = gamma.to(DEV), beta.to(DEV)
    cls_o, reg_o = torch.zeros(N, P, max(n_cls, 1), device=DEV), torch.zeros(N, P, 4, device=DEV)
    gcls_d, greg_d = gcls.to(DEV), greg.to(DEV)
    geo = dict(N=N, H=H, W=W, Cout=C, groups=G, n_cls=n_cls, n_reg=n_reg, P=P, point_off=point_off, cls_stride=max(n_cls, 1), eps=1e-5)
    run_top(make_top(nat.TOP_HEAD_FINAL, off={0: ws.off('raw'), 3: ws.off('stats'), 4: ws.off('stage')},
                     ptr={0: g_d.data_ptr(), 1: b_d.data_ptr(), 2: cls_o.data_ptr(), 3: reg_o.data_ptr()}, **geo), ws)
    run_top(make_top(nat.TOP_HEAD_FINAL_BWD, off={0: ws.off('raw'), 1: ws.off('dact'), 3: ws.off('stats'), 4: ws.off('stage'), 5: ws.off('dstage'), 6: ws.off('dscale')},
                     ptr={0: g_d.data_ptr(), 1: b_d.data_ptr(), 2: gcls_d.data_ptr(), 3: greg_d.data_ptr()}, **geo), ws)
    # torch: t = bf16(relu(gn(raw))) treated as the leaf (the GN backward is tested on its own)
    t = bf16r(F.relu(F.group_norm(raw.permute(0, 2, 1).reshape(N, C, H, W), G, gamma, beta, 1e-5))).reshape(N, C, HW).permute(0, 2, 1)
    t = t.clone().requires_grad_(True)
    wt, bt_, st = wf.clone().requires_grad_(True), bias.clone().requires_grad_(True), torch.tensor(1.3, requires_grad=True)
    sc = torch.cat([torch.ones(n_cls), st.expand(n_reg)]) if n_reg else torch.ones(n_cls)
    out = (t @ wt.t() + bt_) * sc
    up = torch.cat([gcls[:, point_off:point_off + HW, :n_cls], greg[:, point_off:point_off + HW, :n_reg]], -1)
    out.backward(up)
    if n_cls:
        assert rel(cls_o[:, point_off:point_off + HW], out.detach()[..., :n_cls]) < 1e-5
    if n_reg:
        assert rel(reg_o[:, point_off:point_off + HW], out.detach()[..., n_cls:]) < 1e-5
    ds = ws.get('dstage').cpu()
    assert rel(ds[:no * C].view(no, C), wt.grad) < 1e-4
    assert rel(ds[no * C:no * C + no], bt_.grad) < 1e-4
    if n_reg:
        assert rel(ws.get('dscale').cpu(), st.grad.reshape(1)) < 1e-4
    assert rel(ws.get('dact').float(), t.grad) < 6e-3


# ------------------------------------------------------------------------------------------------ weight gradients
WG_CASES = [
    # N, H, W, Cin, Cout, k, s
    (2, 20, 19, 64, 64, 3, 1),
    (1, 33, 17, 64, 64, 3, 2),
    (2, 24, 40, 64, 128, 1, 1),
    (2, 23, 21, 64, 64, 1, 2),
    (1, 18, 24, 128, 128, 3, 1),
    (2, 17, 16, 64, 128, 3, 2),
    (2, 16, 16, 32, 32, 3, 2),
    (1, 40, 24, 32, 64, 1, 1),
    (1, 12, 20, 128, 128, 1, 1),
]


@pytest.mark.parametrize('impl', ['umma', 'simt'])
@pytest.mark.parametrize('case', WG_CASES)
def test_wgrad_matches_autograd(case, impl):
    N, H, W, Cin, Cout, k, s = case
    torch.manual_seed(7)
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
    x = bf16r(torch.randn(N, H, W, Cin))
    dz = bf16r(torch.randn(N, Ho, Wo, Cout))
    ws = Workspace(DEV)
    ws.add('x', x.to(torch.bfloat16))
    ws.add('dz', dz.to(torch.bfloat16))
    ws.add('ds', shape=(k * k, Cin, Cout), dtype=torch.float32)
    ws.finalize()
    run_top(make_top(nat.TOP_WGRAD, N=N, H=H, W=W, Cin=Cin, Ho=Ho, Wo=Wo, Cout=Cout, ksize=k, stride=s,
                     impl=nat.WGRAD_UMMA if impl == 'umma' else nat.WGRAD_SIMT, off={0: ws.off('x'), 1: ws.off('dz'), 5: ws.off('ds')}), ws)
    want = torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2), (Cout, Cin, k, k), dz.permute(0, 3, 1, 2), stride=s, padding=k // 2)
    got = ws.get('ds').cpu().permute(2, 1, 0).reshape(Cout, Cin, k, k)
    assert rel(got, want) < 2e-4, rel(got, want)


@pytest.mark.parametrize('path', ['im2col+umma', 'simt'])
@pytest.mark.parametrize('fmt', ['f32', 'u8'])
def test_wgrad_stem(fmt, path):
    torch.manual_seed(8)
    N, H, W, Cout = 2, 45, 150, 64
    Ho, Wo = conv_out(H, 3, 2), conv_out(W, 3, 2)
    if fmt == 'u8':
        img = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8)
        x = bf16r((img.float() - 127.5) / 127.5).permute(0, 3, 1, 2)
    else:
        img = torch.randn(N, 3, H, W)
        x = bf16r(img)
    dz = bf16r(torch.randn(N, Ho, Wo, Cout))
    ws = Workspace(DEV)
    ws.add('dz', dz.to(torch.bfloat16))
    ws.add('ds', shape=(32, Cout), dtype=torch.float32)          # 27 (tap, ci) rows + 5 padding rows of the tensor-core path
    ws.add('x27', shape=(N, Ho, Wo, 32), dtype=torch.bfloat16)
    ws.finalize()
    offs = {1: ws.off('dz'), 5: ws.off('ds')}
    if path != 'simt':
        offs[0] = ws.off('x27')
    run_top(make_top(nat.TOP_WGRAD_STEM, N=N, H=H, W=W, Cin=3, Ho=Ho, Wo=Wo, Cout=Cout, ksize=3, stride=2, impl=nat.WGRAD_SIMT if path == 'simt' else nat.WGRAD_UMMA,
                     off=offs), ws, input=img.to(DEV).contiguous(), fmt=nat.INPUT_U8_NHWC if fmt == 'u8' else nat.INPUT_F32_NCHW)
    want = torch.nn.grad.conv2d_weight(x, (Cout, 3, 3, 3), dz.permute(0, 3, 1, 2), stride=2, padding=1)
    stage = ws.get('ds').cpu()
    assert float(stage[27:].abs().max()) == 0.0
    got = stage[:27].reshape(9, 3, Cout).permute(2, 1, 0).reshape(Cout, 3, 3, 3)
    assert rel(got, want) < 2e-4, rel(got, want)


# ------------------------------------------------------------------------------------------------ data gradients
@pytest.mark.parametrize('case', [(2, 20, 19, 64, 64, 3, 1), (1, 33, 17, 64, 64, 3, 2), (2, 24, 40, 64, 128, 1, 1), (2, 23, 21, 64, 64, 1, 2),
                                  (1, 18, 24, 128, 128, 3, 1), (2, 17, 16, 64, 128, 3, 2), (2, 16, 16, 32, 32, 3, 2)])
def test_dgrad_is_the_forward_kernel_on_transposed_weights(case):
    """dx = conv_transpose(dz, W): stride 1 = the forward conv of dz with the (ci <-> co swapped, tap-flipped) weights staged by
    PACK_CONV_DGRAD; stride 2 = the same stride-1 conv on the zero-inserted dz (written by NORM_BWD_APPLY in training)."""
    N, H, W, Cin, Cout, k, s = case
    torch.manual_seed(9)
    Ho, Wo = conv_out(H, k, s), conv_out(W, k, s)
    w = bf16r(torch.randn(Cout, Cin, k, k) * 0.1)
    dz = bf16r(torch.randn(N, Ho, Wo, Cout))
    prev = bf16r(torch.randn(N, H, W, Cin))          # an existing gradient the result is accumulated onto
    if s == 2:
        up = torch.zeros(N, H, W, Cout)
        up[:, ::2, ::2, :] = dz
    else:
        up = dz
    q = nat.conv_query(N, H, W, Cout, H, W, Cin, k, 1)
    wd = w.to(DEV)
    ws = Workspace(DEV)
    ws.add('dzu', up.to(torch.bfloat16))
    ws.add('dx', prev.to(torch.bfloat16))
    ws.add('wp', shape=(w.numel(),), dtype=torch.bfloat16)
    ws.finalize()
    d = nat.PackDesc(kind=nat.PACK_CONV_DGRAD, Cout=Cout, Cin=Cin, k=k, cc=q['cc'], n=w.numel(), src=wd.data_ptr(), dst=ws.buf.data_ptr() + ws.off('wp'))
    table = desc_table([d], DEV)
    run_top(make_top(nat.TOP_PACK, n_desc=1, max_n=w.numel(), ptr={0: table.data_ptr()}), ws)
    run_top(make_top(nat.TOP_CONV, N=N, H=H, W=W, Cin=Cout, Ho=H, Wo=W, Cout=Cin, ksize=k, stride=1, cc=q['cc'],
                     off={0: ws.off('dzu'), 1: ws.off('dx'), 2: ws.off('dx'), 4: ws.off('wp')}), ws)
    want = torch.nn.grad.conv2d_input((N, Cin, H, W), w, dz.permute(0, 3, 1, 2), stride=s, padding=k // 2).permute(0, 2, 3, 1) + prev
    got = ws.get('dx').float().cpu()
    assert float((got - want).abs().max()) <= 2.0 ** -7 * float(want.abs().max()) + 1e-5


# ------------------------------------------------------------------------------------------------ optimizer
@pytest.mark.parametrize('max_norm,nesterov', [(10.0, False), (0.5, False), (0.0, True)])
def test_sgd_step_matches_torch(max_norm, nesterov):
    torch.manual_seed(10)
    n = 100003
    p0, g0 = torch.randn(n), torch.randn(n) * 0.01
    pt = torch.nn.Parameter(p0.clone())
    opt = torch.optim.SGD([pt], lr=0.05, momentum=0.9, weight_decay=1e-4, nesterov=nesterov)
    p_d, m_d = p0.clone().to(DEV), torch.zeros(n, device=DEV)
    sq = torch.zeros(1, dtype=torch.float64, device=DEV)
    for step in range(3):
        g = g0 * (step + 1)
        pt.grad = g.clone()
        if max_norm > 0:
            total = torch.nn.utils.clip_grad_norm_([pt], max_norm)
        opt.step()
        g_d = g.clone().to(DEV)
        nat.check(nat.lib().lfd_grad_sqnorm(nat.ptr(g_d), n, nat.ptr(sq), nat.stream_ptr()))
        nat.check(nat.lib().lfd_sgd_step(nat.ptr(p_d), nat.ptr(g_d), nat.ptr(m_d), n, 0.05, 0.9, 0.0, 1e-4, int(nesterov), max_norm, 1.0,
                                         nat.ptr(sq), nat.stream_ptr()))
        torch.cuda.synchronize()
        if max_norm > 0:
            assert abs(float(sq.sqrt()) - float(total)) < 1e-4 * float(total)
            assert torch.allclose(g_d.cpu(), pt.grad, rtol=1e-5, atol=1e-8)
        assert torch.allclose(p_d.cpu(), pt.detach(), rtol=1e-5, atol=1e-6)
