"""Worker of tests/test_gpu_tied.py::test_data_parallel_replicas_stay_identical (one process per GPU, launched by
torch.distributed.run): tiednet replicas, each on its own batch, train 4 steps in bf16 with the NCCL gradient sync; the
parameters must then be bit-identical on every rank (the tie groups' shared slices travel in the bucket of their lowest
edge like any other slice)."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from convnet_b200 import lib  # noqa: E402
from convnet_b200.net import Net, dp_unique_id  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib.load()
    lib.set_precision("bf16")
    net = Net("tiednet", 64, seed=3)
    idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        idt.copy_(torch.frombuffer(bytearray(dp_unique_id()), dtype=torch.uint8))
    dist.broadcast(idt, 0)
    net.dp_init(rank, world, bytes(idt.cpu().numpy().tobytes()), 1 << 18)     # several buckets
    g = torch.Generator(device="cuda").manual_seed(100 + rank)
    net.input_tensor().normal_(generator=g)
    net.labels_tensor().copy_(torch.randint(0, net.num_classes, (64,), device="cuda", generator=g, dtype=torch.int32))
    p0 = net.params_tensor().clone()
    for _ in range(4):
        net.train_step()
    torch.cuda.synchronize()
    p = net.params_tensor().clone()
    gathered = [torch.empty_like(p) for _ in range(world)]
    dist.all_gather(gathered, p)
    res = {"bit_identical_across_ranks": all(torch.equal(gathered[0], x) for x in gathered),
           "max_param_change": float((p - p0).abs().max())}
    if rank == 0:
        print(json.dumps(res), flush=True)
    net.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
