"""The row checker of tests/composed_check.py on the CPU: it accepts the oracle's bf16 emulation against the fp32
oracle, and rejects faults a composition bug makes, naming the row.  Three of them (the first three below) pass the
single global rule of test_gpu_parity.py, which is why the per-row rule exists."""
import pytest
import torch

from oracle import f5_oracle as O
from composed_check import assert_rows, exact_zero_rows, row_errors
from helpers import ocfg_of, rel


def global_rule(got, ref, emu):
    """test_gpu_parity.within_drift over the whole tensor."""
    return rel(got, ref) < min(max(3 * rel(emu, ref), 2e-3), 2e-2)


@pytest.fixture(scope="module")
def gate():
    from f5_tts_mlx_b200.weights import GATE_CONFIG, random_dit_weights
    return ocfg_of(GATE_CONFIG), random_dit_weights(GATE_CONFIG, seed=1234)


def forward(gate, B, N, lens=None, drops=(False, False), seed=0):
    cfg, W = gate
    g = torch.Generator().manual_seed(seed + N)
    x = torch.randn(B, N, 100, generator=g)
    cond = torch.randn(B, N, 100, generator=g) * 2 - 1
    text = torch.randint(0, 2545, (B, 40), generator=g, dtype=torch.int32)
    t = torch.tensor(0.37)
    mask = (torch.arange(N)[None] < torch.tensor(lens)[:, None]) if lens is not None else None
    ref = O.dit_forward(x, cond, text, t, *drops, mask, W, cfg)
    emu = O.dit_forward(x, cond, text, t, *drops, mask, W, cfg, O.Precision(True))
    return ref[None], emu[None]          # one branch


@pytest.fixture(scope="module")
def one(gate):
    return forward(gate, 1, 200)


@pytest.fixture(scope="module")
def two(gate):
    return forward(gate, 2, 300, lens=[300, 211])


def rejects(got, ref, emu, where):
    with pytest.raises(AssertionError) as e:
        assert_rows(got, ref, emu)
    assert "branch %d, utterance %d, frame %d" % where in str(e.value), str(e.value)
    return str(e.value)


def test_accepts_the_emulation(one, two):
    for ref, emu in (one, two):
        rep = assert_rows(emu, ref, emu)
        assert rep.ratio == 1.0
        eg = row_errors(emu, ref)
        assert 1.0 < eg.max() / eg.median() < 2.0          # the bf16 row drift is tight: worst ~1.2-1.3x the median


def test_rejects_the_last_three_frames_scaled(one):
    ref, emu = one
    got = emu.clone()
    got[:, :, -3:] *= 1.05
    assert global_rule(got, ref, emu)
    rejects(got, ref, emu, (0, 0, ref.shape[2] - 3 + int(row_errors(got, ref)[0, 0, -3:].argmax())))


def test_rejects_frame_0_of_the_last_utterance_scaled(two):
    ref, emu = two
    got = emu.clone()
    got[:, 1, 0] *= 1.10
    assert global_rule(got, ref, emu)
    rejects(got, ref, emu, (0, 1, 0))


def test_rejects_eight_rows_offset(one):
    ref, emu = one
    got = emu.clone()
    rows = [5, 17, 63, 64, 100, 127, 128, 190]
    got[:, :, rows] += 0.03 * ref[:, :, rows].abs().mean(-1, keepdim=True)
    assert global_rule(got, ref, emu)
    e = rejects(got, ref, emu, (0, 0, int(row_errors(got, ref)[0, 0].argmax())))
    assert int(row_errors(got, ref)[0, 0].argmax()) in rows, e


def test_rejects_a_one_frame_shift_at_an_utterance_boundary(two):
    """Utterance 1's first row holds the last row of utterance 0 (a flat row index off by one at the boundary)."""
    ref, emu = two
    got = emu.clone()
    got[:, 1, 0] = emu[:, 0, -1]
    rejects(got, ref, emu, (0, 1, 0))


def test_rejects_swapped_cfg_halves(gate):
    """pred + (pred - null) * cfg with pred and null exchanged in utterance 1 only."""
    refp, emup = forward(gate, 2, 150, lens=[150, 97], seed=5)
    refn, emun = forward(gate, 2, 150, lens=[150, 97], drops=(True, True), seed=5)
    cfg = 2.0
    ref, emu = refp + (refp - refn) * cfg, emup + (emup - emun) * cfg
    got = emu.clone()
    got[:, 1] = emun[:, 1] + (emun[:, 1] - emup[:, 1]) * cfg
    e = rejects(got, ref, emu, (0, 1, int(row_errors(got, ref)[0, 1].argmax())))
    assert "utterance 1" in e


def test_per_utterance_rule_and_lens():
    """A fault inside one utterance that the worst-row part sees as small is still caught by its own rel L2; rows past
    `lens` do not count."""
    g = torch.Generator().manual_seed(0)
    ref = torch.randn(2, 3, 50, 16, generator=g)
    emu = ref + 1e-3 * torch.randn(ref.shape, generator=g)
    got = emu.clone()
    got[1, 2] += 4e-3 * torch.randn(50, 16, generator=g)        # every row of (branch 1, utterance 2) ~4x worse
    with pytest.raises(AssertionError, match="branch 1, utterance 2"):
        assert_rows(got, ref, emu, factor=3.0, floor=1.0)        # the floor disables the worst-row part
    bad = emu.clone()
    bad[1, 0, 40:] = 1e3                                          # beyond lens[0] = 40: ignored
    assert assert_rows(bad, ref, emu, lens=[40, 50, 50]).ratio <= 1.0 + 1e-12
    with pytest.raises(AssertionError, match="branch 1, utterance 0, frame 40"):
        assert_rows(bad, ref, emu, lens=[41, 50, 50])


def test_exact_zero_rows_names_the_row():
    buf = torch.zeros(3, 256, 8)
    buf[:, :150] = 1.0
    exact_zero_rows(buf, 150)
    exact_zero_rows(buf, [150, 200, 256])
    buf[2, 201, 5] = 1e-30
    with pytest.raises(AssertionError, match="utterance 2, frame 201"):
        exact_zero_rows(buf, 150)
