"""The persistent two-pass kernel keeps its intermediate in a ring of RING transforms (slot = b % RING).  Any RING >= 2
works, not only powers of two, including a ring shrunk before the launch for a small batch.  Ring size and lag only
change the schedule, not the per-tile arithmetic, so the result must equal the default plan's bit for bit, and every
transform must match the long-double reference within the bounds of tools/emulate.cu."""
import numpy as np
import pytest
import torch

import fourier_b200 as fb
from oracle import oracle as O
from helpers import per_transform_err, poisoned_like, truth_ld

pytestmark = pytest.mark.gpu

NP = {"f32": np.complex64, "f64": np.complex128}
TOL = {"f32": 2e-6, "f64": 5e-15}


def create(real, n):
    return fb.create_fft_f32(n) if real == "f32" else fb.create_fft_f64(n)


@pytest.mark.parametrize("real,n,ring,lag,batch", [
    ("f32", 1 << 20, 3, 2, 7),     # slots wrap at 3
    ("f32", 1 << 20, 3, 1, 1),     # one transform on a 3-slot ring (shrunk to 2)
    ("f64", 1 << 16, 24, 12, 40),
    ("f64", 1 << 16, 5, 3, 2),     # two transforms on a 5-slot ring (shrunk to 2, lag 1)
])
def test_ring_of_any_size(monkeypatch, real, n, ring, lag, batch):
    monkeypatch.setenv("FOURIER_B200_RING", str(ring))
    monkeypatch.setenv("FOURIER_B200_LAG", str(lag))
    p = create(real, n)
    monkeypatch.delenv("FOURIER_B200_RING")
    monkeypatch.delenv("FOURIER_B200_LAG")
    ref = create(real, n)
    assert p.info()["path_name"] == ref.info()["path_name"]
    x = O.fill_input(batch, n, NP[real], first_transform=3)
    xd = torch.from_numpy(x).cuda()
    got, want = poisoned_like(xd), poisoned_like(xd)
    p.transform(xd, got, fb.Transform.Fft)
    ref.transform(xd, want, fb.Transform.Fft)
    torch.cuda.synchronize()
    got, want = got.cpu().numpy(), want.cpu().numpy()
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    err = per_transform_err(got, truth_ld(x, int(fb.Transform.Fft)))
    assert (err < TOL[real]).all(), f"transforms {np.nonzero(~(err < TOL[real]))[0].tolist()} of {batch}: {err}"
    p.close()
    ref.close()
