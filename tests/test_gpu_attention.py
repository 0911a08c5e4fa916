"""YB_OP_ATTENTION (csrc/attention_sm90.cu) alone vs F.scaled_dot_product_attention in fp32 on the same rounded q/k/v.

Tolerance per element: |err| <= tol * (1 + A(|V|)), tol = 2^-9 (f16) / 2^-6 (bf16), where A(|V|) is the fp32 attention
applied to |V| -- the scale on which the rounding of P to f16/bf16 acts.  (1 + |ref|) would be too tight: the
outputs are weighted sums of values of both signs and can cancel."""
import pytest
import torch
import torch.nn.functional as F

from yolort_b200 import _C

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
TOL = {torch.float16: 2.0 ** -9, torch.bfloat16: 2.0 ** -6}


def _desc(qkv_full, in_off, E, out_full, out_off, N, H, W, heads, dtype):
    d = _C.OpDesc()
    d.kind, d.dtype = _C.YB_OP_ATTENTION, _C.dtype_code(dtype)
    d.N, d.H, d.W, d.Cin, d.in_cstride = N, H, W, 3 * E, qkv_full.shape[-1]
    d.in_ = qkv_full.data_ptr() + in_off * 2
    d.Ho, d.Wo, d.Cout, d.out_cstride = H, W, E, out_full.shape[-1]
    d.out = out_full.data_ptr() + out_off * 2
    d.ksize = heads
    return d


def _reference(qkv, N, L, E, heads):
    """qkv: [N, L, 3E] (rounded values, fp32) -> (attention [N, L, E], attention applied to |V|)."""
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    d = E // heads
    q, k, v = (qkv[..., i * E:(i + 1) * E].reshape(N, L, heads, d).transpose(1, 2) for i in range(3))
    ref = F.scaled_dot_product_attention(q, k, v)
    ref_abs = F.scaled_dot_product_attention(q, k, v.abs())
    return (ref.transpose(1, 2).reshape(N, L, E), ref_abs.transpose(1, 2).reshape(N, L, E))


def _run_case(N, H, W, dtype, qk_scale=1.0, heads=4, in_off=0, in_extra=0, out_off=0, out_extra=0, seed=0):
    E = 64 * heads
    L = H * W
    g = torch.Generator().manual_seed(seed)
    full_in = torch.randn(N, H, W, in_off + 3 * E + in_extra, generator=g)
    full_in[..., in_off:in_off + 2 * E] *= qk_scale
    full_in = full_in.to(dtype).to(DEV)
    sentinel = -7.0
    full_out = torch.full((N, H, W, out_off + E + out_extra), sentinel, dtype=dtype, device=DEV)
    d = _desc(full_in, in_off, E, full_out, out_off, N, H, W, heads, dtype)
    _C.Plan([d], DEV).run()
    torch.cuda.synchronize()
    qkv = full_in[..., in_off:in_off + 3 * E].float().reshape(N, L, 3 * E)
    ref, ref_abs = _reference(qkv, N, L, E, heads)
    got = full_out[..., out_off:out_off + E].float().reshape(N, L, E)
    err = (got - ref).abs()
    bad = int((err > TOL[dtype] * (1.0 + ref_abs)).sum())
    assert bad == 0, f"{bad} violations, max err {float(err.max()):.3e} (L={L}, N={N}, {dtype})"
    # the channels around the output window are never written
    if out_off:
        assert torch.all(full_out[..., :out_off] == sentinel)
    if out_extra:
        assert torch.all(full_out[..., out_off + E:] == sentinel)
    return got, full_in, full_out, d, qkv


# (H, W) -> L = 1, 12, 63, 64, 65, 100, 400, 1600, 4096, with the largest batch that keeps the fp32 reference small
SHAPES = [((1, 1), 32), ((3, 4), 32), ((7, 9), 32), ((8, 8), 32), ((5, 13), 32), ((10, 10), 32), ((20, 20), 32),
          ((40, 40), 8), ((64, 64), 2)]


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("hw,N", SHAPES, ids=[f"L{h * w}" for (h, w), _ in SHAPES])
def test_attention_matches_sdpa_in_wider_buffers(hw, N, dtype):
    """qkv at channel offset 8 of a buffer with 24 extra channels; output window at offset 16 of E + 48 channels."""
    _run_case(N, hw[0], hw[1], dtype, in_off=8, in_extra=16, out_off=16, out_extra=32)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("hw,N", [((20, 20), 32), ((13, 20), 4)])
def test_attention_matches_sdpa_dense_views(hw, N, dtype):
    _run_case(N, hw[0], hw[1], dtype)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("regime,qk_scale", [("near_uniform", 0.2), ("peaked", 3.0)])
def test_attention_score_regimes(regime, qk_scale, dtype):
    """Near-uniform weights (every key matters) and strongly peaked ones (logits of +-tens: the running-max
    rescale of the online softmax decides the result)."""
    N, H, W, E = 4, 20, 20, 256
    L = H * W
    _, _, _, _, qkv = _run_case(N, H, W, dtype, qk_scale=qk_scale, seed=5)
    q, k = (qkv[..., i * E:(i + 1) * E].reshape(N, L, 4, 64).transpose(1, 2) for i in range(2))
    logits = (q @ k.transpose(-1, -2)) / 8.0
    p = logits.softmax(-1)
    if regime == "near_uniform":
        ent = float(-(p * p.clamp_min(1e-30).log()).sum(-1).mean())
        assert ent > 0.95 * torch.log(torch.tensor(float(L)))
    else:
        assert float(logits.abs().max()) > 30.0 and float(p.max(-1).values.mean()) > 0.5


def test_attention_two_heads_and_determinism():
    got, full_in, full_out, d, _ = _run_case(3, 9, 15, torch.float16, heads=2, out_off=8, out_extra=8)
    plan = _C.Plan([d], DEV)     # full_in stays alive: the descriptor points into it
    plan.run()
    torch.cuda.synchronize()
    again = full_out[..., 8:8 + 128].float().reshape(3, 135, 128)
    assert torch.equal(got, again)
