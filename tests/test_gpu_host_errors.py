"""A refused call on a live net raises ValueError with the host's reason, and leaves the process and the net able to go
on: each refusal below happens before the call writes anything, so the net trains afterwards.  Each case runs in a
fresh interpreter, so a regression to exit() fails its test instead of ending pytest."""
import pytest

from test_host_errors_cpu import run

pytestmark = pytest.mark.gpu

STEP = """
    import math
    import torch
    from convnet_b200 import net

    def step(n, fill=True):
        if fill:
            n.input_tensor().normal_()
        n.labels_tensor().copy_(torch.randint(0, n.num_classes, (n.batch_size,), device="cuda", dtype=torch.int32))
        loss = n.train_step()
        assert math.isfinite(loss), loss
"""


def test_refused_optimizer_configs():
    out = run(STEP + """
    n = net.Net("tiny+bn", 32, seed=3)
    step(n)
    torch.cuda.synchronize()                             # the update's streams included
    weights, gamma, params = n.optimizer_state(0), n.bn_optimizer_state("conv1"), n.params_tensor().clone()
    try:
        n.set_optimizer(0, weights={"optimizer_type": "LBFGS", "epsilon": 0.01})
    except ValueError as e:
        print("WEIGHTS", e)
    try:
        n.set_bn_optimizer("conv1", gamma={"epsilon": 0.01, "weight_norm_limit": 1.0})
    except ValueError as e:
        print("GAMMA", e)
    assert n.optimizer_state(0) == weights and n.bn_optimizer_state("conv1") == gamma
    assert torch.equal(n.params_tensor(), params)
    step(n)
    assert n.optimizer_state(0)["weights"]["step"] == weights["weights"]["step"] + 1
    print("TRAINS")
    """)
    assert "WEIGHTS" in out and "LBFGS" in out
    assert "GAMMA" in out and "weight_norm_limit" in out
    assert "TRAINS" in out


def test_upload_out_of_range():
    out = run(STEP + """
    n = net.Net("tiny", 32, seed=1)                      # 8 x 12 x 12 inputs
    it = net.DataIterator(32, 8, 16, 12, seed=2)
    images = torch.randn(32, 8, 16, 16).pin_memory()
    try:
        it.upload(images, first=8)
    except ValueError as e:
        print("UPLOAD", e)
    it.upload(images)
    it.get_batch(n)
    step(n, fill=False)
    print("TRAINS")
    """)
    assert "UPLOAD" in out and "outside the chunk" in out
    assert "TRAINS" in out


def test_get_batch_on_a_net_of_another_input_shape():
    out = run(STEP + """
    g = torch.Generator().manual_seed(5)
    images = torch.randn(64, 8, 16, 16, generator=g).pin_memory()
    labels = torch.randint(0, 10, (64,), generator=g, dtype=torch.int32)
    h = net.DataHandler(images, labels, batch_size=32, gpu_image_size=12, translate=True, seed=3)
    other = net.Net("lenet", 32, seed=1)
    try:
        h.get_batch(other)
    except ValueError as e:
        print("SHAPE", e)
    n = net.Net("tiny", 32, seed=1)
    h.get_batch(n)
    assert h.last_indices()["start"] == 0                # the refused call drew no batch
    loss = n.train_step()
    assert math.isfinite(loss), loss
    print("TRAINS")
    """)
    assert "SHAPE" in out and "input layer" in out
    assert "TRAINS" in out
