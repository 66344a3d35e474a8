"""Plans of one size on two GPUs of one process.  Kernel attributes such as the dynamic shared-memory limit belong to a
kernel *and device*: a plan on the second GPU must run after the same kernel already ran on the first, and give the
same bits."""

import numpy as np
import pytest

import fourier_b200 as fb
from helpers import per_transform_err, truth_ld

pytestmark = pytest.mark.gpu

TOL = {"f32": 1e-5, "f64": 1e-12}

# CTA-path sizes ({2,3}-smooth, not a power of two): the kernel's two shared-memory buffers of N complex values each
# exceed the 48 KB of dynamic shared memory a kernel gets without the attribute.
CTA_CASES = [("f32", 6144), ("f64", 3072)]


@pytest.mark.parametrize("prec,n", CTA_CASES)
def test_cta_plan_on_two_devices(prec, n):
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("needs at least 2 GPUs")
    dt = np.complex64 if prec == "f32" else np.complex128
    assert 2 * n * np.dtype(dt).itemsize > 48 * 1024
    rng = np.random.default_rng(n)
    x = (rng.standard_normal((8, n)) + 1j * rng.standard_normal((8, n))).astype(dt)
    outs = []
    try:
        for dev in (0, 1):
            fb.set_device(dev)
            plan = fb.create_fft_f32(n) if prec == "f32" else fb.create_fft_f64(n)
            info = plan.info()
            assert info["path_name"] == "onchip_cta" and info["device"] == dev, info
            with torch.cuda.device(dev):
                xd = torch.from_numpy(x).to(f"cuda:{dev}")
                y = torch.empty_like(xd)
                plan.transform(xd, y, fb.Transform.Fft)
                torch.cuda.synchronize()
            outs.append(y.cpu().numpy())
            plan.close()
    finally:
        fb.set_device(0)
    want = truth_ld(x, 0)
    for dev, y in enumerate(outs):
        err = per_transform_err(y, want).max()
        assert err < TOL[prec], (dev, err)
    assert np.array_equal(outs[0], outs[1])
