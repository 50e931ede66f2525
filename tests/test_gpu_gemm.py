"""GPU: the wgmma GEMM family through the C ABI (vnb_op_gemm) against an fp32 torch contraction of the same bf16
operands, for every fused epilogue, ragged M, more tiles than SMs, and BOTH tile variants: one CTA per 128 x 256 tile
and the CTA pair (a cluster of two vertically adjacent tiles sharing the W tile by TMA multicast; vnb_set_option
"gemm_pair").  Tolerances: outputs are
bf16-rounded (rel 2^-8) or fp32 of a bf16 x bf16 -> fp32 accumulation; the two variants must agree bit for bit."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def L():
    from vampnet_b200 import _lib
    _lib.lib()
    return _lib


@pytest.fixture(params=[0, 1], ids=["single_cta", "cta_pair"])
def pair(request, L):
    prev = L.C.c_int32()
    L.check(L.lib().vnb_get_option(b"gemm_pair", L.C.byref(prev)))
    L.check(L.lib().vnb_set_option(b"gemm_pair", request.param))
    yield request.param
    L.check(L.lib().vnb_set_option(b"gemm_pair", prev.value))


def operands(M, N, K, seed=0):
    g = torch.Generator().manual_seed(seed)
    A = torch.randn(M, K, generator=g).bfloat16().cuda()
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).bfloat16().cuda()
    return A, W, A.float() @ W.float().t(), g


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def run(L, epi, A, W, out, out2=None, bias=None, T=1, Tpad=8):
    M, K = A.shape
    N = W.shape[0]
    L.check(L.lib().vnb_op_gemm(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(out), L.ptr(out2) if out2 is not None else None,
                                L.ptr(bias) if bias is not None else None, T, Tpad, L.stream_ptr()))
    torch.cuda.synchronize()


def close_bf16(got, want):
    err = (got.float() - want).abs()
    tol = 2.0 ** -7 * want.abs() + 2e-3
    assert bool((err <= tol).all()), f"max err {err.max().item():.3e} at {int((err - tol).argmax())}"


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (128, 256, 1280), (256, 512, 128), (300, 512, 256), (1, 256, 64),
                                   (129, 256, 192), (40000, 512, 128), (6144, 1280, 2560)])
def test_bf16_out(L, pair, M, N, K):
    A, W, ref, _ = operands(M, N, K, seed=M + N + K)
    out = torch.full((M, N), float("nan"), device="cuda", dtype=torch.bfloat16)
    run(L, L.EPI_BF16, A, W, out)
    close_bf16(out, ref)


def test_bias_f32_and_resid(L, pair):
    A, W, ref, g = operands(300, 512, 256, seed=1)
    bias = torch.randn(512, generator=g).cuda()
    out = torch.full((300, 512), float("nan"), device="cuda")
    run(L, L.EPI_BIAS_F32, A, W, out, bias=bias)
    assert (out - (ref + bias)).abs().max() < 2e-4
    x0 = torch.randn(300, 512, generator=g).cuda()
    out = x0.clone()
    run(L, L.EPI_RESID, A, W, out)
    assert (out - (x0 + ref)).abs().max() < 2e-4


def test_geglu(L, pair):
    M, N, K = 300, 1024, 256
    A, W, ref, _ = operands(M, N, K, seed=2)
    half = N // 2
    Wi = torch.empty_like(W)  # per 256-row tile: [128 value rows | 128 gate rows]  (include/vampnet_b200.h)
    for t in range(N // 256):
        Wi[t * 256: t * 256 + 128] = W[t * 128:(t + 1) * 128]
        Wi[t * 256 + 128: (t + 1) * 256] = W[half + t * 128: half + (t + 1) * 128]
    out = torch.full((M, half), float("nan"), device="cuda", dtype=torch.bfloat16)
    run(L, L.EPI_GEGLU, A, Wi, out)
    close_bf16(out, ref[:, :half] * gelu_tanh(ref[:, half:]))


@pytest.mark.parametrize("B,T,d", [(4, 75, 256), (2, 200, 256)])
def test_qkv_with_transposed_v(L, pair, B, T, d):
    M, N, K = B * T, 3 * d, 256
    A, W, ref, _ = operands(M, N, K, seed=3)
    Tpad = (T + 7) // 8 * 8
    qk = torch.full((M, 2 * d), float("nan"), device="cuda", dtype=torch.bfloat16)
    vT = torch.zeros((B, d, Tpad), device="cuda", dtype=torch.bfloat16)
    run(L, L.EPI_QKV, A, W, qk, out2=vT, T=T, Tpad=Tpad)
    close_bf16(qk, ref[:, :2 * d])
    close_bf16(vT[:, :, :T], ref[:, 2 * d:].view(B, T, d).permute(0, 2, 1))


def test_variants_agree_bit_for_bit(L):
    """Same operands, same K order per output element: the pair kernel must reproduce the single-CTA kernel exactly
    (so switching the option can never change a generated token)."""
    outs = []
    A, W, _, _ = operands(1000, 1280, 1280, seed=9)
    x0 = torch.randn(1000, 1280, generator=torch.Generator().manual_seed(1)).cuda()
    prev = L.C.c_int32()
    L.check(L.lib().vnb_get_option(b"gemm_pair", L.C.byref(prev)))
    try:
        for p in (0, 1):
            L.check(L.lib().vnb_set_option(b"gemm_pair", p))
            out = x0.clone()
            run(L, L.EPI_RESID, A, W, out)
            outs.append(out)
    finally:
        L.check(L.lib().vnb_set_option(b"gemm_pair", prev.value))
    assert torch.equal(outs[0], outs[1])


def set_opt(L, name, value):
    prev = L.C.c_int32()
    L.check(L.lib().vnb_get_option(name, L.C.byref(prev)))
    L.check(L.lib().vnb_set_option(name, value))
    return prev.value


@pytest.mark.parametrize("M,N,K", [(300, 512, 256), (1, 256, 64), (257, 256, 128), (1000, 1280, 1280),
                                   (40000, 512, 128), (24576, 1280, 1280), (6144, 1280, 2560)])
def test_residual_epilogue_shapes(L, M, N, K):
    """x += A.W^T against fp32 torch and bit for bit between the two tile variants, for ragged M (clipped rows), a
    single row, many tiles per CTA and the benchmark's attention-output / FFN-down shapes."""
    A, W, ref, g = operands(M, N, K, seed=M + K)
    x0 = torch.randn(M, N, generator=g).cuda()
    prev_pair = set_opt(L, b"gemm_pair", 0)
    try:
        outs = []
        for mode in (0, 1):
            L.check(L.lib().vnb_set_option(b"gemm_pair", mode))
            out = x0.clone()
            run(L, L.EPI_RESID, A, W, out)
            outs.append(out)
    finally:
        set_opt(L, b"gemm_pair", prev_pair)
    assert (outs[1] - (x0 + ref)).abs().max() < 2e-4
    assert torch.equal(outs[0], outs[1])


def test_tile_variants_agree_in_the_fused_stack():
    """Through the model: the residual epilogues also write the bf16 copy of the residual stream and the RMSNorm row
    statistics the next GEMM consumes; logits and generated tokens must be bit-identical for both tile variants."""
    from tests.test_gpu_parity import TINY_C2F, TINY_COARSE, build
    from vampnet_b200 import _lib as L
    prev_pair = set_opt(L, b"gemm_pair", 1)
    try:
        for cfgd, C_, T in ((TINY_COARSE, 4, 100), (TINY_C2F, 14, 37)):
            cfg, sd, model, cb, codec = build(cfgd)
            z = torch.randint(0, 1025, (3, C_, T), generator=torch.Generator().manual_seed(T)).cuda()
            kw = dict(start_tokens=z.clamp(max=1023), _sampling_steps=3, seed=1, return_signal=False)
            outs, toks = [], []
            for mode in (1, 0):
                L.check(L.lib().vnb_set_option(b"gemm_pair", mode))
                outs.append(model.forward_codes(z, codec).clone())
                toks.append(model.generate(codec, **kw))   # graphs are cached per option value
            assert torch.equal(outs[0], outs[1]) and torch.equal(toks[0], toks[1])
    finally:
        set_opt(L, b"gemm_pair", prev_pair)


def test_pair_occupancy_reported(L):
    n = L.C.c_int32()
    L.check(L.lib().vnb_get_option(b"gemm_pair_max_clusters", L.C.byref(n)))
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f"co-resident CTA pairs: {n.value} on {sms} SMs")
    assert 0 < n.value <= sms // 2


def test_unknown_option_is_an_error(L):
    with pytest.raises(RuntimeError, match="unknown option"):
        L.check(L.lib().vnb_set_option(b"no_such_option", 1))
