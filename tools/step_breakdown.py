"""Per-call-site kernel times of one full-size eager training step (CUDA events around every libb2d launch; the events
serialise nothing but each launch is timed in isolation from launch gaps).  Usage: python tools/step_breakdown.py [B]
[--ffn]  (--ffn: LoRA on the attention and feed-forward linears instead of the attention set)"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from finetrainers_b200 import ops  # noqa: E402
from finetrainers_b200.model import LORA_FFN_TARGETS, B200LTXTransformer, LTXConfig  # noqa: E402
from finetrainers_b200.trainer import SFTTrainStep  # noqa: E402

ARGS = [a for a in sys.argv[1:] if not a.startswith("--")]
B = int(ARGS[0]) if ARGS else 1
FFN = "--ffn" in sys.argv[1:]
dev = torch.device("cuda", 0)
torch.manual_seed(0)
model = B200LTXTransformer(LTXConfig(), torch.bfloat16, dev)
with torch.no_grad():
    for name, p in model.named_parameters():
        if "scale_shift_table" in name:
            p.normal_(0, 1.0 / p.shape[-1] ** 0.5)
        elif "norm_q" in name or "norm_k" in name:
            p.fill_(1.0)
        else:
            p.normal_(0, 0.02)
model.add_adapter(64, 64, target_modules=list(LORA_FFN_TARGETS) if FFN else None)
with torch.no_grad():
    for name, p in model.named_parameters():
        if "lora_B" in name:
            p.normal_(0, 0.01)
model.prepare()
st = SFTTrainStep(model, use_cuda_graph=False)
lat = torch.randn(B, 128, 7, 16, 24, device=dev).bfloat16()
ehs = (torch.randn(B, 128, 4096, device=dev) * 0.1).bfloat16()
mask = (torch.arange(128, device=dev)[None] < 77).expand(B, 128).contiguous()
mean, std = torch.zeros(B, 128, device=dev), torch.ones(B, 128, device=dev)


def run():
    st.train_step({"encoder_hidden_states": ehs, "encoder_attention_mask": mask},
                  {"latents": lat, "latents_mean": mean, "latents_std": std})


for _ in range(2):
    run()
torch.cuda.synchronize()
ops.TIMING = True
N = 3
for _ in range(N):
    run()
torch.cuda.synchronize()
ops.TIMING = False
t = ops.collect_kernel_times()
tot = sum(v[0] for v in t.values()) / N
print(f"sum of timed launches: {tot:.3f} ms/step")
for k, (ms, n) in sorted(t.items(), key=lambda kv: -kv[1][0]):
    print(f"{k:32s} {ms / N:8.3f} ms/step  {n // N:5d} launches  {1e3 * ms / n:8.1f} us avg")
