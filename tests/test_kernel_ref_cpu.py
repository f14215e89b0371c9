"""oracle/kernel_ref.py on the CPU: emulations of each kernel's arithmetic pass their bounds, emulations with one seeded mistake
fail them, and the exact input constructions of tests/test_kernel_bounds_gpu.py hold their invariants."""
import math
from types import SimpleNamespace

import pytest
import torch

from oracle import kernel_ref as R

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64


def _bits_truncate_bf16(x32: torch.Tensor) -> torch.Tensor:
    return (x32.view(torch.int32) & -65536).view(F32).to(BF16)          # drop the low 16 bits: round toward zero


# ----------------------------------------------------------------------------------------------- GEMM
def _gemm_case(seed=0, M=300, N=192, K=256):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g).to(BF16)
    w = (torch.randn(N, K, generator=g) * K ** -0.5).to(BF16)
    bias = torch.randn(N, generator=g)
    return a, w, bias


def _emulate_gemm(a, w, bias, mistake=None):
    """fp32 accumulation, + bias, round to nearest even (or the seeded mistake)."""
    acc = a.float() @ w.float().t()
    if mistake == "drop_kblock":                  # tile (0, 0) skips its first 64-wide K block
        acc[:128, :64] -= a[:128, :64].float() @ w[:64, :64].float().t()
    x = acc + bias
    if mistake == "truncate":
        return _bits_truncate_bf16(x)
    out = x.to(BF16)
    if mistake == "wrong_row":
        out[77] = (out[77].float() * 1.05).to(BF16)
    return out


@pytest.mark.parametrize("mistake", [None, "truncate", "drop_kblock", "wrong_row"])
def test_gemm_emulation_and_seeded_mistakes(mistake):
    a, w, bias = _gemm_case()
    ref, bound = R.linear_ref(a, w, bias)
    out = _emulate_gemm(a, w, bias, mistake)
    if mistake is None:
        r, f = R.check_rounded(out, ref, bound, BF16, "emulated GEMM", ("row", "col"))
        assert r < 0.75 and f > 0.999, (r, f)
    else:
        with pytest.raises(AssertionError):
            R.check_rounded(out, ref, bound, BF16, f"GEMM with {mistake}", ("row", "col"))


def test_gemm_gelu_emulation_passes():
    a, w, bias = _gemm_case(1)
    ref, bound = R.linear_ref(a, w, bias, act="gelu")
    out = (0.5 * (a.float() @ w.float().t() + bias) * (1 + torch.special.erf((a.float() @ w.float().t() + bias) / math.sqrt(2)))).to(BF16)
    R.check_rounded(out, ref, bound, BF16, "emulated GEMM + GELU")


def test_integer_operands_are_exact():
    """|a|, |b| <= 8 and K <= 4096: every partial sum is an integer below 2^18, so fp32 holds each exactly."""
    for K in (8, 56, 72, 392, 4096):
        a, b = R.int_operands(129, 96, K, seed=K)
        acc, absacc = R.gemm_acc(a, b)
        assert float(absacc.max()) < 2 ** 18
        assert torch.equal((a.float() @ b.float().t()).double(), acc)


def test_tie_values_are_halfway_points():
    for v in (257.0, 259.0, -257.0, 514.0, 1028.0):
        assert bool(R.is_tie(torch.tensor([v], dtype=F64), BF16)), v
    for v in (2049.0, 2051.0, -2049.0, 4098.0):
        assert bool(R.is_tie(torch.tensor([v], dtype=F64), F16)), v
    for v in (256.0, 258.0):
        assert not bool(R.is_tie(torch.tensor([v], dtype=F64), BF16)), v
    for v in (2048.0, 2050.0):
        assert not bool(R.is_tie(torch.tensor([v], dtype=F64), F16)), v
    # round-to-nearest-even of the ties, the values the bit-exact GEMM tests expect
    assert R.round_to(torch.tensor([257.0, 259.0], dtype=F64), BF16).tolist() == [256.0, 260.0]
    assert R.round_to(torch.tensor([2049.0, 2051.0, 7e4, -7e4], dtype=F64), F16).tolist() == [2048.0, 2052.0, 65504.0, -65504.0]


def test_ulp():
    x = torch.tensor([1.0, 1.5, 255.0, 256.0, -3.0, 0.0], dtype=F64)
    assert R.ulp(x, BF16).tolist() == [2 ** -7, 2 ** -7, 1.0, 2.0, 2 ** -6, 2.0 ** -133]
    assert R.ulp(x, F16).tolist()[:4] == [2 ** -10, 2 ** -10, 2 ** -3, 2 ** -2]


# ----------------------------------------------------------------------------------------------- attention
def _rand_attn(B, H, n, seed, peaky=False, spike=None):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(B, H, n, 64, generator=g, dtype=F64) * (1.5 if peaky else 1.0) * (math.log2(math.e) / 8)
    k = torch.randn(B, H, n, 64, generator=g, dtype=F64)
    if peaky:
        k *= torch.linspace(0.2, 6.0, n, dtype=F64)[None, None, :, None]
    if spike is not None:
        q = q * 0.3 + 2.0
        k = k * 0.3
        k[:, :, spike] = 3.0
    v = torch.randn(B, H, n, 64, generator=g, dtype=F64)
    return q.to(BF16), k.to(BF16), v.to(BF16)


@pytest.mark.parametrize("B,H,n,kind", [(1, 2, 300, "random"), (2, 1, 129, "random"), (1, 2, 700, "peaky"), (1, 1, 700, "spike")])
def test_attention_emulation_passes_bound(B, H, n, kind):
    q, k, v = _rand_attn(B, H, n, seed=n, peaky=kind == "peaky", spike=650 if kind == "spike" else None)
    ref, bound = R.attention_ref(q, k, v)
    out = R.emulate_attention(q, k, v)
    r = R.check_bound(out, ref, bound, "emulated attention", ("batch", "row", "col"))
    assert r < 0.75, r


def test_exact_attention_constructions_hold():
    # one-hot codes: distinct, and the target beats every other key by >= 256 in log2 units
    q, k, v, exp = R.onehot_case(1, 2, 300, 300, seed=0)
    s = q.double() @ k.double().transpose(-1, -2)
    top2 = s.topk(2, dim=-1).values
    assert (top2[..., 0] == 128 * 64).all() and (top2[..., 0] - top2[..., 1] >= 256).all()
    for h in range(2):
        assert torch.unique(k[0, h].double(), dim=0).shape[0] == 300
    assert torch.equal(R.emulate_attention(q, k, v), exp)
    # uniform rows: every score -16, every probability 1
    q, k, v, exp = R.uniform_case(2, 1, 200, seed=1)
    s = q.double() @ k.double().transpose(-1, -2)
    assert (s == -16).all() and float(v.double().abs().sum(2).max()) < 2 ** 24
    assert torch.equal(R.emulate_attention(q, k, v), exp)
    # correlated rounding: all the non-zero-v keys' probabilities round down to 0.5 in bf16
    q, k, v, ref = R.rounding_case(1, 2, 300, seed=2)
    p = torch.exp2(torch.tensor(-0.99609375, dtype=F64))
    assert float(R.round_to(p, BF16)) == 0.5 and float((p - 0.5) / p) > 2.5e-3
    assert R.match_fraction(R.emulate_attention(q, k, v), ref, BF16) >= 0.99


ATTN_MISTAKES = ["mask_off_by_one", "skip_alpha", "l_after_round"]


@pytest.mark.parametrize("mistake", ATTN_MISTAKES)
def test_attention_seeded_mistakes_fail(mistake):
    if mistake == "mask_off_by_one":         # one zeroed key joins the softmax of the ragged last tile
        q, k, v, exp = R.uniform_case(1, 2, 300, seed=3)
        assert not torch.equal(R.emulate_attention(q, k, v, mask_extra=1), exp)
    elif mistake == "skip_alpha":            # O is not rescaled when the running maximum grows
        q, k, v, exp = R.onehot_case(1, 2, 300, 300, seed=4)
        assert not torch.equal(R.emulate_attention(q, k, v, skip_alpha=True), exp)
    else:                                    # l summed from the bf16-rounded probabilities
        q, k, v, ref = R.rounding_case(1, 2, 300, seed=5)
        out = R.emulate_attention(q, k, v, l_after_round=True)
        _, bound = R.attention_ref(q, k, v)
        with pytest.raises(AssertionError):
            R.check_rounded(out, ref, bound, BF16, "attention with l after rounding")
    # a missing rescale also breaks the bound of random rows with a late dominant key
    if mistake == "skip_alpha":
        q, k, v = _rand_attn(1, 2, 300, seed=6, spike=290)
        ref, bound = R.attention_ref(q, k, v)
        r, _ = R.bound_ratio(R.emulate_attention(q, k, v, skip_alpha=True), ref, bound)
        assert r > 1.0, r


def test_attention_path_rule_for_132_sms():
    """The restated launch rule on an H100 SXM: which shapes are persistent, split in 2 / 3 / 4, or plain."""
    assert R.attention_path(8, 16, 1374, 1374, 132, True) == ("persistent", 1)
    assert R.attention_path(1, 7, 9000, 9000, 132, True) == ("plain", 1)         # 497 tiles, tail 101: no split
    assert R.attention_path(1, 16, 4 * 1374, 4 * 1374, 132, True) == ("split", 3)  # 688 tiles, tail 28
    assert R.attention_path(2, 16, 4 * 1374, 4 * 1374, 132, True) == ("split", 2)  # 1 376 tiles, tail 56
    assert R.attention_path(1, 16, 4 * 1374, 4 * 1374, 132, False) == ("plain", 1)
    parts = {R.attention_path(1, h, 24 * 128, 24 * 128, 132, True)[1] for h in range(1, 64)}
    assert {2, 3} <= parts


# ----------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("C", [128, 1024, 2048])
@pytest.mark.parametrize("out_dtype", [BF16, F32, F16])
def test_layernorm_emulation_passes_bound(C, out_dtype):
    g = torch.Generator().manual_seed(C)
    x = torch.randn(64, C, generator=g) + 1e3 * torch.randn(64, 1, generator=g)     # common offset 1000 x the spread
    x[:8] = 0.25 + 1e-4 * torch.randn(8, C, generator=g)                              # near-constant rows: eps dominates
    w, b = 1 + 0.1 * torch.randn(C, generator=g), 0.1 * torch.randn(C, generator=g)
    ref, bound = R.layernorm_ref(x, w, b, 1e-5, out_dtype)
    # fp32 emulation: per-lane sums then a butterfly, as the kernel
    xl = x.float().reshape(64, C // 128, 32, 4).permute(0, 2, 1, 3).reshape(64, 32, -1)
    mean = xl.sum(-1).sum(-1, keepdim=True) / C
    d = x.float() - mean
    rstd = torch.rsqrt((d * d).reshape(64, 32, -1).sum(-1).sum(-1, keepdim=True) / C + 1e-5)
    out = (d * rstd * w + b).to(out_dtype)
    R.check_bound(out, ref, bound, "emulated LayerNorm", ("row", "col"))
    # a mean computed in bf16 is far outside it
    bad = ((x.float() - mean.to(BF16).float()) * rstd * w + b).to(out_dtype)
    with pytest.raises(AssertionError):
        R.check_bound(bad, ref, bound, "LayerNorm with a bf16 mean", ("row", "col"))


# ----------------------------------------------------------------------------------------------- camera head
@pytest.mark.parametrize("D,heads,ok", [(768, 8, False), (256, 8, True), (256, 1, True), (2048, 16, True), (1280, 8, False),
                                        (1536, 8, False), (1792, 8, False)])
def test_camera_create_rejects_head_dims_without_a_kernel(D, heads, ok):
    """The camera attention has kernels for head_dim 32, 64, 128 and 256; ovg_camera_create refuses any other head_dim (96, 160,
    192, 224 above), instead of leaving the error to the first forward.  Creation reads no device memory."""
    import ctypes
    from omnivggt_official_b200 import _lib as L
    lib = L.load()
    blocks = (L.BlockWeights * 1)()
    for name, _ in L.BlockWeights._fields_:
        setattr(blocks[0], name, 256)
    cd = L.CameraDesc()
    cd.D, cd.heads, cd.trunk_depth, cd.trunk = D, heads, 1, blocks
    for name, _ in L.CameraDesc._fields_[4:]:
        setattr(cd, name, 256)                       # never dereferenced by create
    h = ctypes.c_void_p()
    rc = lib.ovg_camera_create(ctypes.byref(cd), ctypes.byref(h))
    if ok:
        assert rc == 0, lib.ovg_last_error().decode()
        lib.ovg_camera_destroy(h)
    else:
        assert rc != 0 and "head_dim must be 32, 64, 128 or 256" in lib.ovg_last_error().decode()


def _cam_weights(D, depth, seed):
    g = torch.Generator().manual_seed(seed)

    def r(*s, std=0.02, mean=0.0, bf=False):
        t = torch.randn(*s, generator=g) * std + mean
        return t.to(BF16).float() if bf else t

    blocks = [SimpleNamespace(ln1_w=r(D, std=0.1, mean=1), ln1_b=r(D, std=0.05), w_qkv=r(3 * D, D, std=D ** -0.5, bf=True),
                              b_qkv=r(3 * D, std=0.05), w_proj=r(D, D, std=D ** -0.5, bf=True), b_proj=r(D, std=0.05),
                              g1=r(D, std=0.05, mean=0.25), ln2_w=r(D, std=0.1, mean=1), ln2_b=r(D, std=0.05),
                              w_fc1=r(4 * D, D, std=D ** -0.5, bf=True), b_fc1=r(4 * D, std=0.05),
                              w_fc2=r(D, 4 * D, std=(4 * D) ** -0.5, bf=True), b_fc2=r(D, std=0.05), g2=r(D, std=0.05, mean=0.25))
              for _ in range(depth)]
    return dict(trunk=blocks, tn_w=r(D, std=0.1, mean=1), tn_b=r(D, std=0.05), rn_w=r(D, std=0.1, mean=1), rn_b=r(D, std=0.05),
                empty=r(9, std=0.3), ew=r(D, 9, std=0.3), eb=r(D, std=0.05), mw=r(3 * D, D, std=D ** -0.5, bf=True), mb=r(3 * D, std=0.05),
                f1w=r(D // 2, D, std=D ** -0.5, bf=True), f1b=r(D // 2, std=0.05), f2w=r(9, D // 2, std=(D // 2) ** -0.5),
                f2b=r(9, std=0.05))


@pytest.mark.parametrize("heads", [8, 1])
def test_camera_fp32_emulation_within_tolerance(heads):
    D, B, S = 256, 2, 3
    w = _cam_weights(D, 2, seed=heads)
    tok = torch.randn(B * S, D, generator=torch.Generator().manual_seed(9))
    ref = R.camera_ref(w, tok, B, S, heads)
    emu = R.camera_ref(w, tok, B, S, heads, dtype=F32)
    e = R.camera_error(emu, ref)
    assert e < R.CAM_TOL / 2, e
    # a wrong attention scale (1 / head_dim instead of 1 / sqrt(head_dim)) is far outside it
    bad = R.camera_ref(w, tok, B, S, heads, dtype=F32, attn_scale=1.0 / (D // heads))
    assert R.camera_error(bad, ref) > R.CAM_TOL
