#!/usr/bin/env python
"""ResNet-18 synchronous parameter-server training on N H100s (BASELINE config 2), synthetic data.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_resnet18.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorch_ps_mpi_b200 as ps          # noqa: E402
from pytorch_ps_mpi_b200 import models   # noqa: E402
from pytorch_ps_mpi_b200.ops.preprocess import normalize_nhwc   # noqa: E402

w = ps.runtime.init()
ps.runtime.bind_to_gpu_numa_node(w.device)      # run on the GPU's own socket (what `mpirun --bind-to numa` does)
dev = w.device
torch.backends.cudnn.benchmark = True
torch.manual_seed(0)
model = models.resnet18().to(dev).to(memory_format=torch.channels_last).bfloat16()
opt = ps.SGD(model.named_parameters(), model.parameters(), lr=0.1, momentum=0.9, weight_decay=1e-4,
             code=ps.Identity(), mode="ps", average=True, profile=True)   # engine='device' is picked automatically
model.attach(opt)        # the fused stem kernel acquires the PS broadcast epoch itself: workers queue no wait kernel
gen = torch.Generator().manual_seed(w.rank)
for step in range(50):
    x = torch.randint(0, 256, (256, 3, 224, 224), dtype=torch.uint8, generator=gen).to(dev, non_blocking=True)
    y = torch.randint(0, 1000, (256,), generator=gen).to(dev, non_blocking=True)
    opt.zero_grad(set_to_none=True)
    loss = torch.nn.functional.cross_entropy(model(normalize_nhwc(x)).float(), y)
    loss.backward()
    _, data = opt.step()
    if step % 10 == 0 and w.rank == 0:
        dev_t = {k: f"{v * 1e3:.3f} ms" for k, v in data.items() if k.startswith("dev_")}
        print(f"step {step:3d} loss {loss.item():.3f} engine={data['engine']} {dev_t}")
opt._engine.check()
opt.close()
ps.runtime.shutdown()
