"""Per-launch list of the codec at the north-star's shape (32 ten-second clips, BASELINE.json configs[3]) for
`ncu --profile-from-start off`: one warm encode/decode, then one profiled encode and one profiled decode.

    ncu --profile-from-start off --clock-control none --csv --log-file codec_layers.csv \
        --metrics gpu__time_duration.sum,dram__bytes_read.sum,dram__bytes_write.sum,\
sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_elapsed python tools/codec_layers.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vampnet_b200.codec import DAC  # noqa: E402

B = int(os.environ.get("CODEC_B", "32"))
dev = torch.device("cuda:0")
torch.manual_seed(0)
dac = DAC().to(dev)
x = torch.randn(B, 1, 441600, device=dev) * 0.3
enc = dac.encode(x)
dac.decode(enc["z"])
torch.cuda.synchronize()
torch.cuda.profiler.start()
enc = dac.encode(x)
torch.cuda.synchronize()
y = dac.decode(enc["z"])
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("done", tuple(enc["codes"].shape), tuple(y["audio"].shape if isinstance(y, dict) else y.shape))
