"""Worker of tests/test_gpu_checkpoint.py.
  mode "staging": runs with CONVNET_B200_STAGE_VERIFY=1 (every use of a staged bf16 copy re-converts its fp32 source and
      aborts on a mismatch): a bf16 net with Polyak averaging trains a step after load, after load_polyak_weights and
      after load_current_weights.
  mode "dp" (launched by torch.distributed.run): rank 0 saves after 3 steps, every rank loads into a fresh net and trains
      3 more; the replicas must be bit-identical and equal an uninterrupted run on the same batches."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from convnet_b200 import lib  # noqa: E402
from convnet_b200.net import Net, dp_unique_id, model_text  # noqa: E402


def polyak_model(base, path, after=1, queue=3):
    text = model_text(base).replace("seed: 42\n", "seed: 42\npolyak_after: %d\npolyak_queue_size: %d\n" % (after, queue), 1)
    with open(path, "w") as f:
        f.write(text)
    return path


def staging(tmp):
    assert os.environ.get("CONVNET_B200_STAGE_VERIFY") == "1"
    lib.load()
    lib.set_precision("bf16")
    model = polyak_model(sys.argv[3], os.path.join(tmp, "net.pbtxt"))
    B = 32
    n = Net(model, B, seed=3)
    n.input_tensor().normal_()
    n.labels_tensor().copy_(torch.randint(0, n.num_classes, (B,), device="cuda", dtype=torch.int32))

    def step():
        assert np.isfinite(n.train_step(True))
    for _ in range(2):
        step()
    ckpt = os.path.join(tmp, "a.ckpt")
    n.save(ckpt)
    step()
    n.load(ckpt)
    step()
    for _ in range(2):
        n.polyak_insert()
        step()
    n.load_polyak_weights()
    step()
    n.load_current_weights()
    step()
    n.fprop(False)
    torch.cuda.synchronize()
    n.close()
    print("VERIFY-CHECKPOINT-OK")


def dp():
    import torch.distributed as dist
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib.load()
    lib.set_precision(os.environ.get("DP_PRECISION", "bf16"))
    model, B, ckpt = os.environ.get("DP_MODEL", "lenet"), 32, os.environ["DP_CKPT"]

    def make(seed):
        net = Net(model, B, seed=seed)
        idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            idt.copy_(torch.frombuffer(bytearray(dp_unique_id()), dtype=torch.uint8))
        dist.broadcast(idt, 0)
        net.dp_init(rank, world, bytes(idt.cpu().numpy().tobytes()), 1 << 20)
        return net
    g = torch.Generator(device="cuda").manual_seed(99)
    probe = Net(model, B, seed=7)
    F, classes = probe.input_floats // B, probe.num_classes
    probe.close()
    xg = torch.randn(6, F, world * B, device="cuda", generator=g)
    yg = torch.randint(0, classes, (6, world * B), device="cuda", generator=g, dtype=torch.int32)

    def train(net, steps):
        out = []
        for s in steps:
            net.input_tensor().copy_(xg[s][:, rank * B:(rank + 1) * B].contiguous().view(-1))
            lib.load().convnet_b200_bf16_invalidate(net.input_tensor().data_ptr())   # (a write the library cannot see)
            net.labels_tensor().copy_(yg[s][rank * B:(rank + 1) * B])
            out.append(net.train_step(True))
        torch.cuda.synchronize()
        return out
    whole = make(7)
    train(whole, range(3))
    if rank == 0:
        whole.save(ckpt)
    dist.barrier()
    train(whole, range(3, 6))
    p_whole = whole.params_tensor().clone()
    whole.close()
    resumed = make(11)                             # another seed: the file's decides
    resumed.load(ckpt)
    train(resumed, range(3, 6))
    p = resumed.params_tensor().clone()
    gathered = [torch.empty_like(p) for _ in range(world)]
    dist.all_gather(gathered, p)
    identical = all(torch.equal(gathered[0], t) for t in gathered)
    same = torch.equal(p, p_whole)
    ok = torch.tensor([1 if identical and same else 0], device="cuda")
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    resumed.close()
    if rank == 0:
        print(json.dumps({"ok": ok.item() == 1, "identical_across_ranks": identical, "equal_to_uninterrupted": same}),
              flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok.item() == 1 else 1)


if __name__ == "__main__":
    if sys.argv[1] == "staging":
        staging(sys.argv[2])
    else:
        dp()
