"""The work queue of pair items at f32 2^20 (PairCfg, csrc/fused_kernels.cuh) on the CPU through tools/emulate.cu: every
pair exactly once, every dependency on an earlier queue position, both steady-state gaps; and the queue of one item
per group that FOURIER_B200_PAIR=0 selects.  Asserts the lines are present, so the checks cannot drop out silently."""
from helpers import run_emulator


def test_pair_queue_checked(tmp_path):
    r = run_emulator("emulate", tmp_path)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = r.stdout.splitlines()
    for tag in ("fused work queue f32 2^20, pair items (T1 64, T2 64;", "fused work queue f32 2^20 (FOURIER_B200_PAIR=0)"):
        hit = [line for line in lines if line.startswith(tag)]
        assert len(hit) == 1 and hit[0].endswith("properties OK"), (tag, hit)
