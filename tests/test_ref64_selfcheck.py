"""CPU proof that the fp64 comparators of tests/_ref64.py are tight enough: they accept a correctly rounded fp16 result and reject the same
result with one element moved by 3 ulps, a bias applied one column off, or one 64-wide k-block missing (and, for attention, probabilities
normalised slightly differently or one 64-key block missing).  No GPU: everything here is fp64 on the CPU."""
import pytest
import torch

from _ref64 import check_attn, check_probs, check_tap, gemm_ref, softmax64, ulp16


def rnd(*shape, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def gemm_case(M=96, N=80, K=200):
    a = rnd(M, K, seed=1).half()
    w = rnd(N, K, seed=2, scale=K ** -0.5).half()
    bias = rnd(N, seed=3)
    ref, terms = gemm_ref(a, w, bias=bias)
    return a, w, bias, ref, terms, K + 1


def test_ulp16_binades():
    x = torch.tensor([1.0, 1.5, 0.999, 2.0 ** -14, 2.0 ** -20, 0.0, -3.0, 65504.0], dtype=torch.float64)
    want = torch.tensor([2.0 ** -10, 2.0 ** -10, 2.0 ** -11, 2.0 ** -24, 2.0 ** -24, 2.0 ** -24, 2.0 ** -9, 32.0], dtype=torch.float64)
    assert torch.equal(ulp16(x), want)
    # ulp16 is the spacing of fp16 itself: nextafter in fp16 differs by exactly one ulp16
    h = rnd(1000, seed=9).half()
    nxt = torch.nextafter(h, torch.full_like(h, float("inf")))
    assert torch.equal((nxt.double() - h.double()), ulp16(h.double()))


def test_tap_accepts_correct_rounding():
    _, _, _, ref, terms, k_eff = gemm_case()
    check_tap(ref.half(), ref, terms, k_eff)


@pytest.mark.parametrize("K", [200, 9 * 320])  # 9 * 320: the longest k-loop of the conv edge cases
def test_tap_rejects_3ulp_move(K):
    _, _, _, ref, terms, k_eff = gemm_case(K=K)
    got = ref.half()
    i = int(ref.abs().argmax())
    flat = got.flatten().clone()
    flat[i] = (flat[i].double() + 3 * ulp16(flat[i].double())).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_tap(flat.view_as(got), ref, terms, k_eff)


def test_tap_rejects_bias_one_column_off():
    a, w, bias, ref, terms, k_eff = gemm_case()
    got = (a.double() @ w.double().t() + torch.roll(bias.double(), 1)).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_tap(got, ref, terms, k_eff)


@pytest.mark.parametrize("kb", [0, 1, 3])
def test_tap_rejects_missing_kblock(kb):
    a, w, bias, ref, terms, k_eff = gemm_case()
    keep = torch.ones(a.shape[1], dtype=torch.bool)
    keep[64 * kb:64 * (kb + 1)] = False
    got = (a.double()[:, keep] @ w.double()[:, keep].t() + bias.double()).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_tap(got, ref, terms, k_eff)


def attn_case(S=40, T=200, d=24, qscale=2.0):
    q = rnd(S, d, seed=4, scale=qscale).half()
    k = rnd(T, d, seed=5).half()
    v = rnd(T, d, seed=6).half()
    p = softmax64((q.double() @ k.double().t()) * d ** -0.5)
    return q, k, v, p


def test_attn_accepts_fp16_p_and_exact():
    _, _, v, p = attn_case()
    v64 = v.double()
    check_attn((p @ v64).half(), p, v64)
    check_attn((p.half().double() @ v64).half(), p, v64)
    check_probs(p.half(), p)


def test_attn_rejects_missing_key_block():
    q, k, v, p = attn_case()
    s = (q.double() @ k.double().t()) * q.shape[1] ** -0.5
    s[:, 64:128] = -float("inf")
    got = (softmax64(s) @ v.double()).half()
    with pytest.raises(AssertionError, match="out of bound"):
        check_attn(got, p, v.double())


def test_probs_reject_other_normalisation():
    _, _, _, p = attn_case()
    with pytest.raises(AssertionError, match="out of bound"):
        check_probs((p * (1 + 2.0 ** -9)).half(), p)
    # a sum taken without the last key: every probability a little too large
    q = p.clone()
    q[:, :-1] = p[:, :-1] / p[:, :-1].sum(-1, keepdim=True)
    q[:, -1] = 0
    with pytest.raises(AssertionError, match="out of bound"):
        check_probs(q.half(), p)
