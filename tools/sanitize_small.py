"""Tiny end-to-end run for compute-sanitizer (memcheck / racecheck): every kernel family once at small shapes (the
adapted GEMMs and the LoRA down-projection included), including ragged sizes (T not a multiple of any tile) so that
tail predicates are exercised.  The third model is configuration A of tests/test_gpu_model_configs.py: a 256-entry
vocabulary (2 sampling strips per codebook, mask token 256) with a single predicted codebook."""
import os
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vampnet_b200.codec import DAC  # noqa: E402
from vampnet_b200.modules.transformer import VampNet  # noqa: E402

dev = torch.device("cuda:0")
torch.manual_seed(0)
for cfg in (dict(n_heads=4, n_layers=2, n_codebooks=4, n_conditioning_codebooks=0, embedding_dim=256),
            dict(n_heads=4, n_layers=1, n_codebooks=14, n_conditioning_codebooks=4, embedding_dim=256),
            dict(n_heads=8, n_layers=1, n_codebooks=1, n_conditioning_codebooks=0, embedding_dim=512, vocab_size=256)):
    V = cfg.get("vocab_size", 1024)
    with torch.device(dev):
        m = VampNet(**cfg)
        cb = torch.randn(cfg["n_codebooks"], V, 8)
    codec = types.SimpleNamespace(quantizer=types.SimpleNamespace(
        quantizers=[types.SimpleNamespace(codebook=types.SimpleNamespace(weight=cb[i])) for i in range(cb.shape[0])]))
    for B, T in ((1, 37), (3, 131)):
        z = torch.randint(0, V, (B, cfg["n_codebooks"], T), device=dev)
        mask = torch.ones_like(z)
        mask[:, :, ::5] = 0
        for graph in (False, True):
            m.use_cuda_graph = graph
            # top-p samples from materialised logits (sample_rows_kernel); without it the classifier GEMM's sampling
            # epilogue + sample_combine_kernel run
            for kw in (dict(top_p=0.9), dict(), dict(sample_cutoff=0.5)):
                out = m.generate(codec, start_tokens=z, mask=mask, _sampling_steps=3, return_signal=False, seed=1, **kw)
                assert not (out == V).any()
    m(torch.randn(2, cfg["n_codebooks"] * 8, 19, device=dev))
    # per-request adapters: the LoRA down-projection and the adapted QKV / RESID / GEGLU epilogues, on ragged shapes
    # with base rows and two adapters in one launch (groups of 1 and 2 rows, T = 37 and 131: groups inside tiles)
    sd = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    for i in range(2):
        m.add_adapter(f"a{i}", {**sd, **{k: torch.randn(v.shape) * 0.05 for k, v in sd.items() if ".lora_" in k}})
    for T in (37, 131):
        z = torch.randint(0, V, (4, cfg["n_codebooks"], T), device=dev)
        calls = [dict(start_tokens=z[:1], adapter="a0"), dict(start_tokens=z[1:3]), dict(start_tokens=z[3:], adapter="a1")]
        m.generate_many(codec, [dict(c, _sampling_steps=2, seed=1, return_signal=False) for c in calls])
        m.forward_codes(z, codec, adapter="a1")
for prec in ("tc", "fp32"):
    dac = DAC(encoder_dim=32, decoder_dim=512, precision=prec).to(dev)
    x = torch.randn(2, 1, 768 * 3, device=dev) * 0.3
    enc = dac.encode(x)
    dac.decode(enc["z"])
    dac.quantizer.from_latents(enc["latents"])
    dac.quantizer.from_codes(enc["codes"])
torch.cuda.synchronize()
print("sanitize workload done")
