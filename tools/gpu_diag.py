"""Development diagnostic (not a test, not product): run ONE kernel family on the GPU and print error
statistics against a plain torch computation.  Run each stage in its own process so that a trapping kernel
cannot poison the others.

    python tools/gpu_diag.py <stage>      stage in: gemm_small gemm_epi gemm_big attention codec attention_b32
"""
import math
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vampnet_b200 import _lib as L  # noqa: E402

dev = torch.device("cuda:0")
torch.backends.cuda.matmul.allow_tf32 = False


def stats(name, got, ref):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    print(f"  {name}: max_abs_err={err.max().item():.4e} mean_abs_err={err.mean().item():.4e} "
          f"ref_absmean={ref.abs().mean().item():.4e} nan={int(torch.isnan(got).sum())} "
          f"frac>1e-2={(err > 1e-2 * (1 + ref.abs())).float().mean().item():.4f}", flush=True)
    return err


def bf(x):
    return x.to(torch.bfloat16)


def gelu_tanh(x):
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def run_gemm(M, N, K, epi, T=None, seed=0, check_ref_kernel=False, timing=False):
    lib = L.lib()
    g = torch.Generator(device="cpu").manual_seed(seed)
    A = bf(torch.randn(M, K, generator=g)).to(dev)
    W = bf(torch.randn(N, K, generator=g) / math.sqrt(K)).to(dev)
    ref = A.float() @ W.float().t()
    st = L.stream_ptr()
    print(f"gemm M={M} N={N} K={K} epi={epi}", flush=True)
    if epi == L.EPI_BF16:
        out = torch.full((M, N), float("nan"), device=dev, dtype=torch.bfloat16)
        L.check(lib.vnb_op_gemm(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(out), None, None, 1, 8, st))
        torch.cuda.synchronize()
        err = stats("bf16 out", out, ref)
        if err.max() > 0.1:
            bad = (err > 0.1).nonzero()
            print("   first bad idx:", bad[:8].tolist(), "rows bad:", bad[:, 0].unique()[:16].tolist(),
                  "cols bad:", bad[:, 1].unique()[:16].tolist())
    elif epi == L.EPI_BIAS_F32:
        bias = torch.randn(N, generator=g).to(dev)
        out = torch.full((M, N), float("nan"), device=dev)
        L.check(lib.vnb_op_gemm(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(out), None, L.ptr(bias), 1, 8, st))
        torch.cuda.synchronize()
        stats("f32+bias out", out, ref + bias)
    elif epi == L.EPI_RESID:
        x0 = torch.randn(M, N, generator=g).to(dev)
        out = x0.clone()
        L.check(lib.vnb_op_gemm(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(out), None, None, 1, 8, st))
        torch.cuda.synchronize()
        stats("resid out", out, x0 + ref)
    elif epi == L.EPI_GEGLU:
        # weights arrive interleaved per 256-row tile: [128 value | 128 gate]
        half = N // 2
        Wv, Wg = W[:half], W[half:]
        Wi = torch.empty_like(W)
        for t in range(N // 256):
            Wi[t * 256: t * 256 + 128] = Wv[t * 128:(t + 1) * 128]
            Wi[t * 256 + 128: (t + 1) * 256] = Wg[t * 128:(t + 1) * 128]
        out = torch.full((M, half), float("nan"), device=dev, dtype=torch.bfloat16)
        L.check(lib.vnb_op_gemm(epi, L.ptr(A), L.ptr(Wi), M, N, K, L.ptr(out), None, None, 1, 8, st))
        torch.cuda.synchronize()
        stats("geglu out", out, ref[:, :half] * gelu_tanh(ref[:, half:]))
    elif epi == L.EPI_QKV:
        B = M // T
        d = N // 3
        Tpad = (T + 7) // 8 * 8
        qk = torch.full((M, 2 * d), float("nan"), device=dev, dtype=torch.bfloat16)
        vT = torch.zeros((B, d, Tpad), device=dev, dtype=torch.bfloat16)
        L.check(lib.vnb_op_gemm(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(qk), L.ptr(vT), None, T, Tpad, st))
        torch.cuda.synchronize()
        stats("qk out", qk, ref[:, :2 * d])
        stats("vT out", vT[:, :, :T], ref[:, 2 * d:].view(B, T, d).permute(0, 2, 1))
    if check_ref_kernel:
        o2 = torch.empty(M, N, device=dev)
        L.check(lib.vnb_dbg_gemm_ref(L.ptr(A), L.ptr(W), M, N, K, L.ptr(o2), st))
        torch.cuda.synchronize()
        stats("simt ref kernel", o2, ref)
    if timing and epi == L.EPI_BF16:
        out = torch.empty((M, N), device=dev, dtype=torch.bfloat16)
        for _ in range(3):
            lib.vnb_op_gemm(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(out), None, None, 1, 8, st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        n = 20
        for _ in range(n):
            lib.vnb_op_gemm(epi, L.ptr(A), L.ptr(W), M, N, K, L.ptr(out), None, None, 1, 8, st)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        print(f"  timing: {ms * 1e3:.1f} us  {2.0 * M * N * K / ms / 1e9:.1f} TFLOP/s (includes plan build on host)")
        t0 = time.time()
        for _ in range(n):
            r = A @ W.t()
        torch.cuda.synchronize()
        e0.record()
        for _ in range(n):
            r = A @ W.t()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        print(f"  cublas bf16 : {ms * 1e3:.1f} us  {2.0 * M * N * K / ms / 1e9:.1f} TFLOP/s")


def attention_ref(q, k, v, rel, sat, H):
    """bf16-operand reference (matches oracle 'bf16' mode).  q,k,v: (B,T,d) bf16 cuda."""
    B, T, d = q.shape
    qf = q.float().view(B, T, H, 64).permute(0, 2, 1, 3)
    kf = k.float().view(B, T, H, 64).permute(0, 2, 1, 3)
    vf = v.float().view(B, T, H, 64).permute(0, 2, 1, 3)
    s = qf @ kf.transpose(-1, -2) * 0.125
    idx = (torch.arange(T, device=q.device)[None, :] - torch.arange(T, device=q.device)[:, None]).clamp(-sat, sat) + sat
    bias = rel[idx]  # (T, T, H)
    s = s + bias.permute(2, 0, 1)[None]
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m)
    o = (e.to(torch.bfloat16).float() @ vf) / e.sum(-1, keepdim=True)
    return o.permute(0, 2, 1, 3).reshape(B, T, d)


def run_attention(B, T, H, seed=0, timing=False):
    lib = L.lib()
    d = H * 64
    sat = 128
    g = torch.Generator(device="cpu").manual_seed(seed)
    q = bf(torch.randn(B, T, d, generator=g)).to(dev)
    k = bf(torch.randn(B, T, d, generator=g)).to(dev)
    v = bf(torch.randn(B, T, d, generator=g)).to(dev)
    rel = (torch.randn(2 * sat + 1, H, generator=g) * 0.5).to(dev)
    rel[:36] = rel[36]      # saturate like the real table does beyond |rel| >= 91
    rel[-36:] = rel[-37]
    Tpad = (T + 7) // 8 * 8
    qk = torch.cat([q, k], dim=-1).contiguous()
    vT = torch.zeros(B, d, Tpad, device=dev, dtype=torch.bfloat16)
    vT[:, :, :T] = v.permute(0, 2, 1)
    out = torch.full((B, T, d), float("nan"), device=dev, dtype=torch.bfloat16)
    print(f"attention B={B} T={T} H={H}", flush=True)
    L.check(lib.vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, Tpad, H, L.stream_ptr()))
    torch.cuda.synchronize()
    ref = attention_ref(q, k, v, rel, sat, H)
    err = stats("attn out", out, ref)
    if err.max() > 0.05:
        e2 = err.view(B, T, H, 64)
        print("   per-head max err:", e2.amax(dim=(0, 1, 3)).tolist()[:8])
        print("   per-qtile max err:", [e2[:, i:i + 128].max().item() for i in range(0, T, 128)][:12])
    if timing:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            lib.vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, Tpad, H, L.stream_ptr())
        e0.record()
        n = 20
        for _ in range(n):
            lib.vnb_op_attention(L.ptr(qk), L.ptr(vT), L.ptr(out), L.ptr(rel), sat, B, T, Tpad, H, L.stream_ptr())
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / n
        print(f"  timing: {ms * 1e3:.1f} us  {4.0 * B * H * T * T * 64 / ms / 1e9:.1f} TFLOP/s")


def main():
    stage = sys.argv[1]
    print(f"=== stage {stage} on {torch.cuda.get_device_name(0)}", flush=True)
    if stage == "gemm_small":
        run_gemm(128, 256, 64, L.EPI_BF16, check_ref_kernel=True)
        run_gemm(128, 256, 256, L.EPI_BF16)
        run_gemm(128, 256, 1280, L.EPI_BF16)
        run_gemm(256, 512, 128, L.EPI_BF16)
        run_gemm(300, 512, 256, L.EPI_BF16)
        run_gemm(40000, 512, 128, L.EPI_BF16)  # 313 x 2 tiles: more CTAs than SMs
    elif stage == "gemm_epi":
        run_gemm(300, 512, 256, L.EPI_BIAS_F32)
        run_gemm(300, 512, 256, L.EPI_RESID)
        run_gemm(300, 1024, 256, L.EPI_GEGLU)
        run_gemm(4 * 75, 768, 256, L.EPI_QKV, T=75)
    elif stage == "gemm_big":
        run_gemm(6144, 3840, 1280, L.EPI_BF16, timing=True)
        run_gemm(6144, 1280, 1280, L.EPI_BF16, timing=True)
        run_gemm(6144, 1280, 2560, L.EPI_BF16, timing=True)
        run_gemm(24576, 5120, 1280, L.EPI_BF16, timing=True)
        run_gemm(6144, 5120, 1280, L.EPI_GEGLU)
        run_gemm(8 * 768, 3840, 1280, L.EPI_QKV, T=768)
    elif stage == "attention":
        run_attention(1, 64, 1)
        run_attention(1, 128, 2)
        run_attention(2, 200, 4)
        run_attention(2, 575, 4)
        run_attention(8, 768, 20, timing=True)
        run_attention(2, 3072, 20, timing=True)
    elif stage == "codec":
        sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
        from oracle import dac_oracle as do
        from vampnet_b200.codec import DAC
        cfg = do.CodecConfig()
        prec = sys.argv[2] if len(sys.argv) > 2 else "tc"
        m = DAC(precision=prec)
        m.load_flat(do.make_codec_weights(cfg, seed=0))
        m = m.to(dev)
        print("precision", prec)
        for B in ((1,) if len(sys.argv) > 3 else (1, 4)):
            x = torch.randn(B, 1, 441600, device=dev) * 0.3
            for _ in range(2):
                enc = m.encode(x)
                out = m.decode(enc["z"])
            torch.cuda.synchronize()
            e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            e0.record()
            enc = m.encode(x)
            e1.record()
            out = m.decode(enc["z"])
            e2.record()
            torch.cuda.synchronize()
            te, td = e0.elapsed_time(e1), e1.elapsed_time(e2)
            print(f"codec B={B}: encode {te:.1f} ms ({0.612 * B / te * 1e3:.1f} TFLOP/s)  decode {td:.1f} ms "
                  f"({1.369 * B / td * 1e3:.1f} TFLOP/s)  -> {B * 10.0 / ((te + td) * 1e-3):.1f}x real time", flush=True)
    elif stage == "attention_b32":
        run_attention(32, 768, 20, timing=True)
    else:
        raise SystemExit("unknown stage")
    print("=== done", flush=True)


if __name__ == "__main__":
    main()
