"""The complex-double fused z + y stage fed by asynchronous copies against its register-fed form (DFFT_ZY_FEED=0): the same
per-line arithmetic on the same inputs, so the outputs are bit-identical — forward, inverse and scaled inverse, both
instantiated lengths."""
import os

import pytest

import distributedfft_b200 as dfft

from test_zy_fused import _plan


def _run(plan, out, x, direction, feed):
    import torch

    before = os.environ.get("DFFT_ZY_FEED")
    os.environ["DFFT_ZY_FEED"] = str(feed)  # read by the launcher at every exec
    try:
        plan.execC2C(out, x, direction)
        torch.cuda.synchronize()
    finally:
        if before is None:
            del os.environ["DFFT_ZY_FEED"]
        else:
            os.environ["DFFT_ZY_FEED"] = before
    assert plan.lastLaunchCount() == 2


@pytest.mark.gpu
@pytest.mark.parametrize("shape,prec", [((512, 512, 512), dfft.F64), ((1024, 256, 256), dfft.F64)])
def test_fed_matches_register_fed(shape, prec):
    import torch

    rdt = torch.float64 if prec == dfft.F64 else torch.float32
    g = torch.Generator(device="cuda").manual_seed(23)
    x = torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt), torch.rand(shape, generator=g, device="cuda", dtype=rdt))
    plan = _plan(shape, prec)
    a = torch.empty_like(x)
    b = torch.empty_like(x)
    # With DFFT_ZY_FEED=1, complex-double views on 16-byte aligned buffers always run the fed kernel: an aligned view the
    # copies cannot address fails the exec instead of falling back (launch_zy_fused), so a passing exec here was fed.
    assert all(t.data_ptr() % 16 == 0 for t in (x, a, b))
    for direction, scale in ((dfft.FORWARD, 1.0), (dfft.INVERSE, 1.0), (dfft.INVERSE, 0.125)):
        plan.setScale(1.0, scale)
        _run(plan, a, x, direction, 1)
        _run(plan, b, x, direction, 0)
        assert torch.equal(a, b), f"direction {direction}, scale {scale}: max |diff| {float((a - b).abs().max())}"
        # repeated execs switching between the kernels, on a new input: both draw from the same counters, and an exec that
        # read the previous exec's intermediate would not match
        x2 = torch.complex(torch.rand(shape, generator=g, device="cuda", dtype=rdt), torch.rand(shape, generator=g, device="cuda", dtype=rdt))
        _run(plan, b, x2, direction, 0)
        _run(plan, a, x2, direction, 1)
        assert torch.equal(a, b), f"direction {direction}, scale {scale}, second input: max |diff| {float((a - b).abs().max())}"
        _run(plan, a, x, direction, 1)
        _run(plan, b, x, direction, 0)
        assert torch.equal(a, b), f"direction {direction}, scale {scale}, first input again: max |diff| {float((a - b).abs().max())}"
        del x2
    plan.destroy()
    del x, a, b
    torch.cuda.empty_cache()

