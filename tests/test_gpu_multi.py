"""2-GPU test of the product's data-parallel path (ADVICE round 1): the replacement modules under (a) the package's flat
NCCL all-reduce and (b) torch DistributedDataParallel reproduce the single-process gradient of the concatenated batch.
Needs two visible GPUs; skipped on a single-GPU machine."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _model(etb, cfg):
    import torch.nn as nn

    class HotPath(nn.Module):
        def __init__(self):
            super().__init__()
            e, d, q = cfg["encoder"], cfg["decoder"], cfg["quantizer"]
            self.encoder = etb.ViTEncoder(cfg["image_size"], cfg["patch_size"], **e)
            self.decoder = etb.ViTDecoder(cfg["image_size"], cfg["patch_size"], **d)
            self.quantizer = etb.VectorQuantizer(**q)
            self.pre_quant = etb.QuantLinear(e["dim"], q["embed_dim"])
            self.post_quant = etb.QuantLinear(q["embed_dim"], d["dim"])

        def forward(self, x):
            quant, qloss, _ = self.quantizer(self.pre_quant(self.encoder(x)))
            return ((self.decoder(self.post_quant(quant)) - x) ** 2).mean() + qloss
    return HotPath()


def _worker(rank, world, port, q, use_ddp):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    import enhancing_transformers_b200 as etb
    from enhancing_transformers_b200.configs import CONFIGS
    etb.set_precision("parity")                       # fp32-grade arithmetic: differences are reduction order only
    cfg = CONFIGS["tiny"]
    torch.manual_seed(0)
    model = _model(etb, cfg).cuda()
    imgs = torch.rand(4, 3, 64, 64, generator=torch.Generator().manual_seed(1)).cuda()
    shard = imgs[rank * 2:(rank + 1) * 2]
    if use_ddp:
        net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[rank])
        net(shard).backward()
    else:
        model(shard).backward()
        etb.allreduce_gradients(model.parameters())
    grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    if rank == 0:
        torch.manual_seed(0)
        single = _model(etb, cfg).cuda()
        single(imgs).backward()
        worst = 0.0
        for n, p in single.named_parameters():
            if p.grad is None:
                continue
            worst = max(worst, ((grads[n] - p.grad).norm() / p.grad.norm().clamp_min(1e-30)).item())
        q.put(worst)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("use_ddp", [False, True], ids=["flat_allreduce", "torch_ddp"])
def test_two_gpu_gradients_equal_single_process(use_ddp):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q, use_ddp)) for r in range(2)]
    for p in procs:
        p.start()
    worst = q.get(timeout=240)
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    # the codebook gradient sees different per-rank code sets summed in a different order; everything else is ~1e-6
    assert worst < 1e-4, worst
