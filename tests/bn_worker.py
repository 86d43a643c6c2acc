"""Worker of tests/test_gpu_batchnorm.py.
  mode "twin" (under CONVNET_B200_STAGE_VERIFY=1, where every look-up of a staged bf16 copy re-converts the fp32 tensor and
        aborts on a mismatch): the bf16 twins cnb_bn_apply and cnb_bn_backward emit equal the rounded fp32 results;
  mode "dp" (launched by torch.distributed.run, one process per GPU): after 3 training steps of a "+bn" model on
        different per-rank batches, every parameter, gamma and beta included, is bit-identical across the replicas.
        (Batch statistics are per rank, so there is no 1-rank run on the concatenated batch to compare with.)"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from convnet_b200 import lib  # noqa: E402
from convnet_b200.net import Net, dp_unique_id  # noqa: E402

mode = sys.argv[1]
if mode == "twin":
    assert os.environ.get("CONVNET_B200_STAGE_VERIFY") == "1"
    L = lib.load()
    lib.set_precision("bf16")
    g = torch.Generator(device="cuda").manual_seed(5)
    for n, C in ((128, 4096), (32 * 55 * 55, 16), (100 * 25 * 25, 48), (6 * 5 * 5, 3)):
        x = torch.randn(C * n, device="cuda", generator=g)
        y, d = torch.empty_like(x), torch.randn(C * n, device="cuda", generator=g)
        gamma, beta = torch.rand(C, device="cuda", generator=g) + 0.5, torch.randn(C, device="cuda", generator=g)
        st = torch.zeros(4 * C, device="cuda")
        mu, sg = st[:C], st[C:2 * C]
        gg, gb = torch.empty(C, device="cuda"), torch.empty(C, device="cuda")
        L.cnb_bn_stats(x.data_ptr(), n, C, 1e-5, 0.9, mu.data_ptr(), sg.data_ptr(), None, None)
        for relu in (0, 1):
            L.convnet_b200_emit_bf16_next()
            L.cnb_bn_apply(x.data_ptr(), y.data_ptr(), n, C, gamma.data_ptr(), beta.data_ptr(), mu.data_ptr(), sg.data_ptr(), relu)
            assert L.convnet_b200_bf16_is_staged(y.data_ptr(), C * n) == 1, (n, C, relu)
        for train in (1, 0):
            L.convnet_b200_emit_bf16_next()
            L.cnb_bn_backward(d.data_ptr(), x.data_ptr(), n, C, gamma.data_ptr(), mu.data_ptr(), sg.data_ptr(), train,
                              gg.data_ptr(), gb.data_ptr())
            assert L.convnet_b200_bf16_is_staged(d.data_ptr(), C * n) == 1, (n, C, train)
        torch.cuda.synchronize()
    print("BN-TWIN-OK")
elif mode == "dp":
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    import torch.distributed as dist
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib.load()
    lib.set_precision("bf16")
    model, B = sys.argv[2], int(sys.argv[3])
    net = Net(model, B, seed=7)
    idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        idt.copy_(torch.frombuffer(bytearray(dp_unique_id()), dtype=torch.uint8))
    dist.broadcast(idt, 0)
    net.dp_init(rank, world, bytes(idt.cpu().numpy().tobytes()), 4096)
    g = torch.Generator(device="cuda").manual_seed(100 + rank)               # a different batch on every rank
    p0 = net.params_tensor().clone()
    for _ in range(3):
        net.input_tensor().normal_(generator=g)
        net.labels_tensor().copy_(torch.randint(0, net.num_classes, (B,), device="cuda", generator=g, dtype=torch.int32))
        net.train_step(False)
    torch.cuda.synchronize()
    p = net.params_tensor().clone()
    gathered = [torch.empty_like(p) for _ in range(world)]
    dist.all_gather(gathered, p)
    gammas_moved = all(not torch.equal(p[o:o + c], p0[o:o + c]) for _, _, c, o in net.bn_layers())
    res = {"identical": all(torch.equal(gathered[0], t) for t in gathered), "gammas_moved": gammas_moved}
    if rank == 0:
        print(json.dumps(res), flush=True)
    net.close()
    dist.destroy_process_group()
