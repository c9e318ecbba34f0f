"""The margin-softmax heads (csrc/heads.cu) against the fp64 references of heads_ref.py.

vdk_head_forward / vdk_head_backward are called directly, so that cos_saved, row_lse, logits and both gradients are all
visible; every output sits in a NaN-guarded buffer with a tail (kernel_ref.Guarded), so a store past B x C or an unwritten
element shows.  The autograd surface (margin_ce_loss, head(...)) is checked against the same references.  Each check prints its
worst err / bound ratio (BOUND lines) and the contractions' RMS factors (HEADS lines).
"""
import ctypes as C
import math

import pytest
import torch

import heads_ref as R
from kernel_ref import Guarded
from test_heads_bounds_cpu import CASE, CASE_RMS, GRAD_OUT, HEAD, KINDS

pytestmark = pytest.mark.gpu


def desc_of(h, B, D, Cn):
    from visiondk_b200 import _lib
    d = _lib.HeadDesc()
    d.kind = R.KIND[h["kind"]]
    d.batch, d.feat_dim, d.num_class = B, D, Cn
    d.margin_arc, d.margin_am, d.scale = h["margin_arc"], h["margin_am"], h["scale"]
    d.margin, d.gamma, d.label_smooth = h["margin"], h["gamma"], h["label_smooth"]
    d.mv_weight, d.is_am = h["mv_weight"], int(h["is_am"])
    return d


def run_kernel(lib, feats, w, labels, h, grad_out=1.0, dlogits=None, backward=True):
    """One forward (with logits and cos_saved) and, if asked, one backward (fused, or un-fused with `dlogits`)."""
    from visiondk_b200 import _lib
    B, D = feats.shape
    Cn = w.shape[1]
    d = desc_of(h, B, D, Cn)
    f, wc, y = feats.cuda().contiguous(), w.cuda().contiguous(), labels.cuda().contiguous()
    ws = torch.empty(lib.vdk_head_workspace_bytes(C.byref(d)), dtype=torch.uint8, device="cuda")
    g = dict(logits=Guarded(B, Cn, Cn, torch.float32), cos=Guarded(B, Cn, Cn, torch.float32),
             row_lse=Guarded(1, B, B, torch.float32), loss=Guarded(1, 1, 1, torch.float32))
    _lib.check(lib.vdk_head_forward(C.byref(d), f.data_ptr(), wc.data_ptr(), y.data_ptr(), g["logits"].ptr(), g["loss"].ptr(),
                                    g["row_lse"].ptr(), g["cos"].ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr()),
               "vdk_head_forward")
    out = dict(cos=g["cos"].view, logits=g["logits"].view, row_lse=g["row_lse"].view[0], loss=g["loss"].view[0, 0])
    if backward:
        g["dfeats"], g["dweight"] = Guarded(B, D, D, torch.float32), Guarded(D, Cn, Cn, torch.float32)
        gout = torch.tensor([grad_out], dtype=torch.float32, device="cuda")
        dl = dlogits.cuda().float().contiguous() if dlogits is not None else None
        _lib.check(lib.vdk_head_backward(C.byref(d), f.data_ptr(), wc.data_ptr(), y.data_ptr(),
                                         0 if dl is not None else g["row_lse"].ptr(), 0 if dl is not None else gout.data_ptr(),
                                         dl.data_ptr() if dl is not None else 0, g["dfeats"].ptr(), g["dweight"].ptr(),
                                         ws.data_ptr(), ws.numel(), _lib.stream_ptr()), "vdk_head_backward")
        out.update(dfeats=g["dfeats"].view, dweight=g["dweight"].view)
    torch.cuda.synchronize()
    for name, buf in g.items():
        assert not buf.guard_errors(), f"{name}: {buf.guard_errors()}"
    return out


def check(lib, feats, w, labels, h, grad_out=1.0, dlogits=None, stats=None, tag="", backward=True):
    out = run_kernel(lib, feats, w, labels, h, grad_out, dlogits, backward)
    info = R.check_head(out, feats, w, labels, h, grad_out, dlogits, stats, tag)
    if info["nan_rows"]:   # MV-Softmax (arc) with the label cos > 1: NaN loss, exactly as in the reference
        assert math.isnan(float(out["loss"]))
    return out, info


@pytest.mark.parametrize("case", [CASE, CASE_RMS], ids=["D128", "D16"])
def test_self_test_case_on_gpu(lib, case):
    """The inputs on which test_heads_bounds_cpu.py shows that every listed defect falls outside the bounds.  At D = 16 some
    label cosines of the crafted parallel rows exceed 1: with a product instead of a select for the clamp derivative their
    gradients are NaN.  (At D = 128 the H100's accumulator lands them just below 1.)"""
    feats, w, labels = R.make_case(**case)
    h = R.head_consts(**HEAD)
    out, info = check(lib, feats, w, labels, h, GRAD_OUT, tag=" self-test case")
    if case is CASE_RMS:
        assert info["cos_gt_1"] > 0, "no label cosine above 1: the clamp case is not exercised"
    gt1 = (out["cos"][torch.arange(len(labels)), labels.cuda()] > 1).cpu()
    assert bool(torch.isfinite(out["dfeats"][gt1.cuda()]).all()), "NaN gradients where the label cos exceeds 1"
    assert bool(torch.isfinite(out["dweight"][:, labels[gt1].cuda()]).all()), "NaN gradients where the label cos exceeds 1"


SHAPES = [(1, 64, 2), (7, 8, 9), (8, 16, 255), (160, 128, 256), (257, 512, 257), (160, 64, 1000), (7, 512, 1000), (8, 128, 9)]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"B{b}-D{d}-C{c}" for b, d, c in SHAPES])
@pytest.mark.parametrize("k", range(len(KINDS)))
def test_heads_match_fp64(lib, k, shape):
    B, D, Cn = shape
    stats = {}
    mv_arc = KINDS[k]["kind"] == "mv_softmax" and not KINDS[k]["is_am"]
    for smooth, same in ((0.0, False), (0.1, False), (0.1, True)):
        # MV-Softmax arc: the crafted label rows stop at cos 0.9999 (above 1 its loss is NaN: test_mv_arc_label_cos_above_one)
        feats, w, labels = R.make_case(B, D, Cn, seed=1000 * k + B + D + Cn, same_label=same,
                                       label_cos_max=0.9999 if mv_arc else None)
        h = R.head_consts(**KINDS[k], label_smooth=smooth)
        _, info = check(lib, feats, w, labels, h, grad_out=1.0, stats=stats, tag=f" {h['kind']} {shape} eps={smooth} same={same}")
        assert info["nan_rows"] == 0


def test_mv_arc_label_cos_above_one(lib):
    """MV-Softmax arc with features parallel to their class column: where the kernel's label cos exceeds 1, sqrt(1 - gt^2) is
    NaN and so is the loss, exactly as in the reference.  The un-fused backward is NaN only in those rows and label columns;
    everything else is checked."""
    B, D, Cn = 128, 16, 300
    g = torch.Generator().manual_seed(77)
    w = torch.empty(D, Cn).uniform_(-1, 1, generator=g).renorm(2, 1, 1e-5).mul(1e5)
    labels = torch.randint(0, Cn, (B,), generator=g)
    feats = w[:, labels].t() * torch.empty(B, 1).uniform_(0.05, 20.0, generator=g)
    k = next(i for i, kw in enumerate(KINDS) if kw["kind"] == "mv_softmax" and not kw["is_am"])
    h = R.head_consts(**KINDS[k], label_smooth=0.1)
    out, info = check(lib, feats, w, labels, h, backward=False, tag=" mv-arc gt > 1")
    assert info["nan_rows"] > 0 and math.isnan(float(out["loss"]))
    dl = torch.randn(B, Cn, generator=g)
    check(lib, feats, w, labels, R.head_consts(**KINDS[k]), dlogits=dl, tag=" mv-arc gt > 1 un-fused")


@pytest.mark.parametrize("D", [128, 512])
def test_long_k_contraction(lib, D):
    """dF~ = dcos' . W^T at the face config (C = 58 671, K = 6 * 58 672) in the un-fused backward with random dlogits, where
    dcos = dlogits dz carries a couple of roundings and nothing cancels: the dfeats RMS factor is the contraction's own
    accuracy (heads_ref.KAPPA_DFEATS).  One wgmma chain over this K drifts (test_heads_bounds_cpu.py::
    test_long_k_contraction_needs_the_slabs); heads.cu splits it into fixed-order split-K slabs."""
    B, Cn = 160, 58671
    feats, w, labels = R.make_case(B, D, Cn, seed=58671 + D)
    dl = torch.randn(B, Cn, generator=torch.Generator().manual_seed(D))
    h = R.head_consts(**KINDS[0])
    out = run_kernel(lib, feats, w, labels, h, dlogits=dl)
    R.check_head(out, feats, w, labels, h, dlogits=dl, tag=f" long-K un-fused D={D}", rms_dfeats=True)


@pytest.mark.parametrize("k", [0, 2, 4])
def test_face_config_scale(lib, k):
    """configs/faceX/face.yaml: C = 58 671, B = 160, feat_dim 128: dF~ is one wgmma chain over K = 6 * 58 672."""
    feats, w, labels = R.make_case(160, 128, 58671, seed=58671 + k)
    h = R.head_consts(**KINDS[k], label_smooth=0.1)
    check(lib, feats, w, labels, h, grad_out=1.0, tag=f" face-config {h['kind']}")


def test_face_config_wide_features(lib):
    feats, w, labels = R.make_case(160, 512, 58671, seed=7)
    h = R.head_consts(**KINDS[0], label_smooth=0.1)
    check(lib, feats, w, labels, h, grad_out=1.0, tag=" face-config D=512")


@pytest.mark.parametrize("grad_out", [1.0, 0.37, 1024.0])
def test_fused_backward_scales_with_grad_out(lib, grad_out):
    feats, w, labels = R.make_case(64, 128, 1000, seed=3)
    h = R.head_consts(**KINDS[1], label_smooth=0.1)
    check(lib, feats, w, labels, h, grad_out=R.f32(grad_out), tag=f" grad_out={grad_out}")


@pytest.mark.parametrize("k", range(len(KINDS)))
def test_unfused_backward_with_arbitrary_dlogits(lib, k):
    feats, w, labels = R.make_case(33, 64, 300, seed=40 + k)
    dl = torch.randn(33, 300, generator=torch.Generator().manual_seed(k)) * 3.0
    h = R.head_consts(**KINDS[k])
    check(lib, feats, w, labels, h, dlogits=dl, tag=f" un-fused {h['kind']}")


def _head(k, D, Cn, w):
    from visiondk_b200.heads import ArcFace, CircleLoss, MV_Softmax
    kw = {kk: v for kk, v in KINDS[k].items() if kk != "kind"}
    kind = KINDS[k]["kind"]
    head = (ArcFace(D, Cn, kw["margin_arc"], kw["margin_am"], kw["scale"]) if kind == "arcface" else
            CircleLoss(D, Cn, kw["margin"], kw["gamma"]) if kind == "circleloss" else
            MV_Softmax(D, Cn, kw["is_am"], kw["margin"], kw["mv_weight"], kw["scale"])).cuda()
    with torch.no_grad():
        head.weight.copy_(w)
    return head


@pytest.mark.parametrize("k", [0, 2, 5])
def test_autograd_surface(lib, k):
    """(margin_ce_loss * s).backward() for s in {1, 0.37, 1024} and (head(f, y) * R).sum().backward() against the references,
    at the cosines the ctypes forward reports (the autograd path runs the same kernels)."""
    from visiondk_b200.heads import margin_ce_loss
    B, D, Cn = 48, 128, 700
    feats, w, labels = R.make_case(B, D, Cn, seed=90 + k)
    h = R.head_consts(**KINDS[k], label_smooth=0.1)
    ref = run_kernel(lib, feats, w, labels, h, backward=False)
    head = _head(k, D, Cn, w)
    for s in (1.0, 0.37, 1024.0):
        f = feats.cuda().requires_grad_(True)
        head.weight.grad = None
        loss = margin_ce_loss(head, f, labels.cuda(), 0.1)
        (loss * s).backward()
        out = dict(cos=ref["cos"], loss=loss.detach(), dfeats=f.grad, dweight=head.weight.grad)
        R.check_head(out, feats, w, labels, h, grad_out=R.f32(s), tag=f" autograd fused x{s}")
    Rm = torch.randn(B, Cn, generator=torch.Generator().manual_seed(k)).cuda()
    h0 = R.head_consts(**KINDS[k])
    f = feats.cuda().requires_grad_(True)
    head.weight.grad = None
    logits = head(f, labels.cuda())
    (logits * Rm).sum().backward()
    out = dict(cos=ref["cos"], logits=logits.detach(), dfeats=f.grad, dweight=head.weight.grad)
    R.check_head(out, feats, w, labels, h0, dlogits=Rm.cpu(), tag=" autograd un-fused")


def test_two_forwards_give_identical_cosines(lib):
    """The backward recomputes cos and relies on the forward's row_lse fitting it."""
    feats, w, labels = R.make_case(160, 128, 5000, seed=9)
    h = R.head_consts(**KINDS[0])
    a = run_kernel(lib, feats, w, labels, h, backward=False)["cos"].clone()
    b = run_kernel(lib, feats, w, labels, h, backward=False)["cos"]
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("D", [7, 100])
def test_forward_at_any_feat_dim_and_backward_refusal(lib, D):
    from visiondk_b200 import _lib
    from visiondk_b200.heads import margin_ce_loss
    feats, w, labels = R.make_case(20, D, 50, seed=D)
    h = R.head_consts(**KINDS[0], label_smooth=0.1)
    check(lib, feats, w, labels, h, backward=False, tag=f" forward D={D}")
    B, Cn = 20, 50
    d = desc_of(h, B, D, Cn)
    ws = torch.empty(lib.vdk_head_workspace_bytes(C.byref(d)), dtype=torch.uint8, device="cuda")
    f, wc, y = feats.cuda(), w.cuda(), labels.cuda()
    lse, gout = torch.zeros(B, device="cuda"), torch.ones(1, device="cuda")
    df, dw = torch.empty(B, D, device="cuda"), torch.empty(D, Cn, device="cuda")
    rc = lib.vdk_head_backward(C.byref(d), f.data_ptr(), wc.data_ptr(), y.data_ptr(), lse.data_ptr(), gout.data_ptr(), 0,
                               df.data_ptr(), dw.data_ptr(), ws.data_ptr(), ws.numel(), _lib.stream_ptr())
    assert rc != 0 and "multiple of 8" in _lib.last_error()
    head = _head(0, D, Cn, w)
    fr = f.clone().requires_grad_(True)
    loss = margin_ce_loss(head, fr, y, 0.1)
    with pytest.raises(ValueError, match="multiple of 8"):
        loss.backward()
