"""The tile-by-tile check of tests/attn_online_emul.py on the CPU, at 60 s (N = 5625, two utterances, two heads): it
accepts what the FP8 attention kernel may legitimately write, and rejects small faults of the online softmax, naming
where.  fp8_attention_bound (the float64-softmax bound of test_gpu_fp8_attention.py) accepts the first two faults."""
import re

import pytest
import torch

import attn_online_emul as M

B, N, H = 2, 5625, 2
OUT = "e4m3_scaled"


def emulate(ops, kv, **kw):
    O, beta = M.online_softmax(*ops, kv, "fp8", **kw)
    return O, beta, M.expected_output(O, OUT)


@pytest.fixture(scope="module")
def random_case():
    qkv = M.make_qkv("random", B, N, H, seed=3)
    kv = torch.tensor([N, M.KV_LEN[N]])
    ops = M.operands(qkv, B, N, H, "fp8", kv)
    M.assert_exact_logits(ops[0], ops[2], "fp8")
    return ops, kv, emulate(ops, kv)


@pytest.fixture(scope="module")
def tail_last_case():
    qkv = M.make_qkv("tail_last", B, N, H, seed=4)
    kv = torch.tensor([N, M.KV_LEN[N]])
    ops = M.operands(qkv, B, N, H, "fp8", kv)
    M.assert_exact_logits(ops[0], ops[2], "fp8")
    return ops, kv, emulate(ops, kv)


def accepts(got, case):
    O, beta, _ = case[2]
    return M.check_output(got[0], O, beta, OUT, got[1], what="accepted")


def rejects(got, case, utt=None, head=None):
    """The check fails and names an (utterance, head, q-tile, row) where got's code is one O within beta cannot give."""
    O, beta, _ = case[2]
    with pytest.raises(AssertionError) as e:
        M.check_output(got[0], O, beta, OUT, got[1], what="fault")
    msg = str(e.value)
    loc = re.search(r"\(utterance (\d+), head (\d+), q-tile (\d+), row (\d+)", msg)
    assert loc, msg
    b, h, t, n = (int(i) for i in loc.groups())
    assert t == n // M.TILE and (utt is None or b == utt) and (head is None or h == head), msg
    print(msg)
    return b, h, n


def old_bound_accepts(got, case):
    """fp8_attention_bound plus the block-scaled output rounding, as test_fp8_attention_random_within_bound applies it."""
    from kernel_check import E4M3_SUB, U_E4M3
    from test_gpu_fp8_attention import fp8_attention_bound
    (qc, sq, kc, sk, vc, sv), kv = case[0], case[1]
    rep = lambda s: s.repeat_interleave(M.TILE, -1)[..., :N, None]
    q, k, v = qc * sq[..., None], kc * rep(sk), vc * rep(sv)
    worst = 0.0
    for h in range(H):
        o, b = fp8_attention_bound(q[:, h:h + 1], k[:, h:h + 1], v[:, h:h + 1], kv)
        bound = b + U_E4M3 * (o.abs() + b) + E4M3_SUB * got[1][:, h:h + 1, :, None]
        worst = max(worst, ((got[0][:, h:h + 1] * got[1][:, h:h + 1, :, None] - o).abs() / bound).max().item())
    print(f"fp8_attention_bound: worst err/bound {worst:.3f}")
    return worst <= 1.0


def test_accepts_the_emulation_in_another_summation_order(random_case):
    ops, kv, _ = random_case
    accepts(emulate(ops, kv, reverse=True)[2], random_case)


def test_accepts_p_rounded_the_other_way_wherever_ambiguous(random_case):
    """With exact logits e takes few distinct values per row (its argument depends only on s - m), so few P are within
    fp32 rounding of an e4m3 boundary: the count is printed."""
    ops, kv, (O, beta, want) = random_case
    O2, _, got = emulate(ops, kv, flip=True)
    print(f"P flipped: O changed in {int((O2 != O).sum())} elements")
    accepts(got, random_case)


@pytest.mark.parametrize("case", ["random", "tail_last"])
def test_accepts_every_error_source_at_its_bound(case, random_case, tail_last_case):
    """P from e (1 +- d), sc, l and the P V accumulation each moved by its full bound (online_softmax(perturb=)): the
    output moves by a large part of beta and is still accepted."""
    c = random_case if case == "random" else tail_last_case
    ops, kv, (O, beta, _) = c
    O2, _, got = emulate(ops, kv, perturb=torch.Generator().manual_seed(11))
    moved = ((O2 - O).abs() / beta).max().item()
    print(f"{case}: perturbed O moved by up to {moved:.2f} beta")
    assert moved > 0.5
    accepts(got, c)


def test_rejects_every_output_times_1_01(random_case):
    O = random_case[2][0]
    got = M.expected_output(O * 1.01, OUT)
    rejects(got, random_case)
    assert old_bound_accepts(got, random_case)


def test_rejects_one_tiles_v_scale_times_1_03(random_case):
    (qc, sq, kc, sk, vc, sv), kv, _ = random_case
    sv2 = sv.clone()
    sv2[1, 0, 17] *= 1.03
    got = emulate((qc, sq, kc, sk, vc, sv2), kv)[2]
    rejects(got, random_case, utt=1, head=0)
    assert old_bound_accepts(got, random_case)


def test_rejects_the_last_partial_tile_dropped(random_case):
    ops, kv, _ = random_case
    kv2 = kv.clone()
    kv2[1] = kv[1] // M.TILE * M.TILE
    assert kv2[1] < kv[1]
    rejects(emulate(ops, kv2)[2], random_case, utt=1)


def test_rejects_two_keys_swapped_inside_a_32_key_group_of_v(random_case):
    (qc, sq, kc, sk, vc, sv), kv, (O, beta, _) = random_case
    s = qc[0, 1, :1] @ kc[0, 1].T                               # the key row 0 of (utterance 0, head 1) weighs most
    key = int(s.argmax())
    vc2 = vc.clone()
    vc2[0, 1, [key, key ^ 1]] = vc[0, 1, [key ^ 1, key]]
    assert not torch.equal(vc2, vc)
    O2, _, got = emulate((qc, sq, kc, sk, vc2, sv), kv)
    b, h, n = rejects(got, random_case, utt=0, head=1)
    assert (O2[b, h, n] - O[b, h, n]).abs().max() > 0


def test_rejects_p_against_the_final_max_when_the_max_arrives_last(tail_last_case):
    """5624 keys 9 ... 14 below a dominant key in the last tile: against the running max their P~ are normal e4m3
    values, against the final max most are below the e4m3 floor.  (On a ramp rising by about 3 logits per tile the two
    differ by less than beta: each tile weighs e^-3 of the next, and its P~ differ only in their 2^-4 rounding.)"""
    ops, kv, _ = tail_last_case
    rejects(emulate(ops, kv, final_max=True)[2], tail_last_case)


def test_rejects_l_summing_the_rounded_p(random_case):
    ops, kv, _ = random_case
    rejects(emulate(ops, kv, l_rounded=True)[2], random_case)
