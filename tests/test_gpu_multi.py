"""GPU, 2 ranks over NCCL (skipped on a single-GPU box): the FSDP-2 path (per-block bf16 all-gather prefetched on a
communication stream, fp32 reduce-scatter of the flat LoRA gradient, sharded AdamW, in-place all-gather of the masters)
produces the same training trajectory as the DDP path (one all-reduce + replicated AdamW), and the all-gathered block
weights drive the same forward loss."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_WORKER = r'''
import os, sys, torch, torch.distributed as dist
sys.path.insert(0, os.environ["B2D_ROOT"]); sys.path.insert(0, os.path.join(os.environ["B2D_ROOT"], "tests"))
from finetrainers_b200.parallel import B200ParallelBackend
from finetrainers_b200.trainer import SFTTrainStep
from _util import build_pair, SMALL
mode = sys.argv[1]
be = B200ParallelBackend(backend="nccl", **({"dp_shards": 2} if mode == "fsdp" else {}))
r = be.rank
O, om, bm = build_pair(dict(SMALL, num_layers=4), 64, seed=3, device=f"cuda:{be.local_rank}")
if mode == "fsdp":
    be.apply_fsdp2(bm, param_dtype=torch.bfloat16, reduce_dtype=torch.float32, output_dtype=None, pp_enabled=False,
                   cpu_offload=False, device_mesh=be.get_mesh()[("dp_shard_cp",)])
    assert bm._fsdp is not None and bm._blk_flat is None
else:
    be.apply_ddp(bm, be.get_mesh())
st = SFTTrainStep(bm, flow_weighting_scheme="none", lr=1e-3, seed=5, use_cuda_graph=(mode == "ddp_graph"),
                  ddp_chunks=(1 if mode == "ddp_serial" else 2))
assert len(st._segments) == (2 if mode in ("ddp", "ddp_graph") else 1)
st.spec.first_frame_conditioning_p = 0.0
losses = []
for i in range(6 if mode == "ddp_graph" else 4):    # graph mode: 2 eager warm-ups, capture, replays
    batch = O.make_synthetic_batch(om.cfg, 2, 2, 4, 9, text_len=24, seed=900 + 10 * i + r, text_scale=1.0)   # rank-specific data
    dev = f"cuda:{be.local_rank}"
    cond = {"encoder_hidden_states": batch["encoder_hidden_states"].to(dev), "encoder_attention_mask": batch["encoder_attention_mask"].to(dev)}
    lat = {"latents": batch["latents"].to(dev), "latents_mean": batch["latents_mean"].to(dev), "latents_std": batch["latents_std"].to(dev)}
    m = st.train_step(cond, lat, sigmas=batch["sigmas"].view(-1).to(dev), noise=batch["noise"].to(dev), sync_metrics=True)
    losses.append((m["train/global_avg_loss"], m["train/global_max_loss"], m["train/grad_norm"]))
torch.cuda.synchronize()
# replicas hold identical adapters after every exchange
mine = bm.lora_flat.clone()
other = [torch.empty_like(mine) for _ in range(2)]
dist.all_gather(other, mine)
assert torch.equal(other[0], other[1]), "ranks diverged"
if r == 0:
    torch.save({"losses": losses, "lora": mine.cpu(), "gathers": (bm._fsdp.blocks.gathers if mode == "fsdp" else 0)}, os.environ["B2D_OUT"] + f".{mode}")
be.wait_for_everyone()
be.destroy()
print("MULTI_OK", mode, r)
'''


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.timeout(600)
def test_fsdp2_matches_ddp_over_nccl(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER)
    out = str(tmp_path / "res")
    env = dict(os.environ, B2D_ROOT=ROOT, B2D_OUT=out, MASTER_ADDR="127.0.0.1", NCCL_DEBUG="WARN")
    for mode, port in (("ddp", "29551"), ("fsdp", "29552"), ("ddp_serial", "29553"), ("ddp_graph", "29554")):
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                            "--master-addr", "127.0.0.1", "--master-port", port, str(script), mode], env=env,
                           capture_output=True, text=True, timeout=280)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
        assert r.stdout.count("MULTI_OK") == 2
    a, b = torch.load(out + ".ddp"), torch.load(out + ".fsdp")
    for (la, ma, ga), (lb, mb, gb) in zip(a["losses"], b["losses"]):
        assert abs(la - lb) / abs(la) < 1e-4 and abs(ma - mb) / abs(ma) < 1e-4 and abs(ga - gb) / abs(ga) < 1e-3
    # same reduction, same AdamW: only the order of the fp32 gradient sum differs (all-reduce vs reduce-scatter)
    assert (a["lora"] - b["lora"]).abs().max().item() < 2e-5
    # the overlapped exchange (two block ranges, all-reduced behind their backward segments) is the serial exchange,
    # and the segment graphs replay what the eager segments compute
    c, d = torch.load(out + ".ddp_serial"), torch.load(out + ".ddp_graph")
    assert (a["lora"] - c["lora"]).abs().max().item() < 1e-6
    for (la, ma, ga), (lc, mc, gc), (ld, md, gd) in zip(a["losses"], c["losses"], d["losses"]):
        assert abs(la - lc) / abs(la) < 1e-6 and abs(ga - gc) / abs(ga) < 1e-5
        assert abs(la - ld) / abs(la) < 1e-5 and abs(ga - gd) / abs(ga) < 1e-4
    # 4 blocks: forward gathers 0..3, backward re-gathers 1, 0 (3 and 2 stay resident); the next step finds 0 and 1 resident
    assert b["gathers"] == 4 + 2 + 3 * (2 + 2)
