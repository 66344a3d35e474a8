"""Pair items of the persistent two-pass kernel at f32 2^20 (PairCfg in csrc/fused_kernels.cuh): one producer lane per
CTA claims two adjacent tiles, one per consumer group.  Each group computes its tile exactly as with one item per group
(FOURIER_B200_PAIR=0), so the outputs must be bit-identical to that configuration, for every transform of a batch that
wraps the L2 ring, at the small batches that shrink the ring, in every direction and scaling, and from host buffers.
Outputs start as NaN and a decoy call on other input runs first, as in test_gpu_persistent_schedule.py."""
import numpy as np
import pytest
import torch

import fourier_b200 as fb
from helpers import poisoned_like, truth_ld
from test_gpu_persistent_schedule import (DECOY, FIRST, check_bits, check_reference, device_input, host_input,
                                          make_plan, run)

pytestmark = pytest.mark.gpu

T = fb.Transform
N = 1 << 20
RING = 4   # the default ring at 2^20 (32 MB / 8 MB)


def plans(monkeypatch):
    monkeypatch.delenv("FOURIER_B200_PAIR", raising=False)
    paired = make_plan(monkeypatch, "f32", N)
    single = make_plan(monkeypatch, "f32", N, FOURIER_B200_PAIR=0)
    assert paired.kernel_name() == single.kernel_name()
    return paired, single


@pytest.mark.parametrize("batch", [1, 2, 3, 5, 11])
@pytest.mark.parametrize("code", [T.Fft, T.Ifft, T.UnscaledIfft, T.SqrtScaledFft])
def test_pairs_bit_identical_to_single_items(monkeypatch, batch, code):
    paired, single = plans(monkeypatch)
    x = device_input("f32", batch, N, FIRST)
    decoy = device_input("f32", batch, N, DECOY)
    want = run(single, x, code, decoy)
    got = run(paired, x, code, decoy)
    torch.cuda.synchronize()
    fail = check_bits(got, want, "f32", RING, f"pairs vs single items, batch {batch}, {code.name}")
    assert fail is None, fail
    if batch == 11 and code in (T.Fft, T.Ifft):   # odd, wraps the ring twice: also against long double
        xh = x.cpu().numpy()
        _, fail = check_reference(got.cpu().numpy(), truth_ld(xh, int(code)), "f32", RING, f"pairs, {code.name}")
        assert fail is None, fail


def test_pairs_from_host_buffers(monkeypatch):
    paired, single = plans(monkeypatch)
    batch = 5
    x = device_input("f32", batch, N, FIRST)
    xh = host_input("f32", batch, N, FIRST, x)
    yh = poisoned_like(xh)
    paired.transform(xh, yh, T.Fft)
    want = run(single, x, T.Fft)
    torch.cuda.synchronize()
    assert np.array_equal(yh.view(np.uint8), want.cpu().numpy().view(np.uint8))
