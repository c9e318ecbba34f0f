"""The training step's depthwise backward (vdk_dwconv7_bwd): the data gradient and the weight gradient from one pass over
the output gradient, each element against the fp64 references and rounding bounds of the two separate entry points
(kernel_ref.py), at the four ConvNeXt-B stage shapes of the bench's batch and at ragged tiles and channel chunks."""
import pytest
import torch

from kernel_ref import (Guarded, check_within, describe_wgrad, dwconv7_bwd_data_bound, dwconv7_reference, wgrad_bound,
                        wgrad_launch, wgrad_reference)
from visiondk_b200 import _lib

pytestmark = pytest.mark.gpu
STATS = {}

# (B, H, W, C): ConvNeXt-B stages at batch 128, ragged tiles with a masked chunk, runtime T below 7
CASES = [(128, 56, 56, 128), (128, 28, 28, 256), (128, 14, 14, 512), (128, 7, 7, 1024), (64, 13, 19, 200), (6, 5, 5, 136)]


@pytest.mark.parametrize("B,H,W,C", CASES, ids=[f"{c[3]}x{c[1]}x{c[2]}b{c[0]}" for c in CASES])
def test_dwconv7_bwd_both_halves_elementwise(lib, B, H, W, C):
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator(device="cuda").manual_seed(B * 5 + C)
    x = torch.randn(B, H, W, C, device="cuda", generator=gen).to(torch.bfloat16)
    g = torch.randn(B, H, W, C, device="cuda", generator=gen).to(torch.bfloat16)
    add = torch.randn(B, H, W, C, device="cuda", generator=gen).to(torch.bfloat16)
    w49 = 0.2 * torch.randn(49, C, device="cuda", generator=gen)
    dx = Guarded(B * H * W, C, C, torch.bfloat16, extra_rows=0, tail=4096)
    dw = Guarded(49, C, C, torch.float32, extra_rows=1, tail=64)
    db = Guarded(1, C, C, torch.float32, extra_rows=1, tail=64)
    dw_init = torch.randn(49, C, device="cuda", generator=gen)
    db_init = torch.randn(1, C, device="cuda", generator=gen)
    dw.fill_(dw_init)
    db.fill_(db_init)
    _lib.check(lib.vdk_dwconv7_bwd(x.data_ptr(), g.data_ptr(), B, H, W, C, w49.data_ptr(), add.data_ptr(), dx.ptr(), dw.ptr(),
                                   db.ptr(), _lib.stream_ptr()), "dwconv7_bwd")
    torch.cuda.synchronize()
    tag = f"dwconv7_bwd {B}x{H}x{W}x{C}"
    ref, mag = dwconv7_reference(g, w49)
    ref += add.double()
    check_within(dx.view.view(B, H, W, C), ref, dwconv7_bwd_data_bound(ref, mag, add), tag + " dx",
                 lambda bad: f"(b, y, x) {bad.any(-1).nonzero()[:6].tolist()}", STATS)
    wref, wmag, bref, bmag = wgrad_reference(x, g)
    WL = wgrad_launch(B, H, W, C, sm)
    check_within(dw.view, dw_init.double() + wref, wgrad_bound(wmag, dw_init, WL), tag + " dw",
                 lambda bad: describe_wgrad(bad, WL), STATS)
    check_within(db.view, db_init.double() + bref[None], wgrad_bound(bmag[None], db_init, WL), tag + " dbias",
                 lambda bad: describe_wgrad(bad, WL), STATS)
    for name, buf in (("dx", dx), ("dw49", dw), ("dbias", db)):
        assert not buf.guard_errors(), f"{name}: " + buf.guard_errors()
