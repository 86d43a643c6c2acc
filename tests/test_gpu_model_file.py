"""Nets built from model files on the GPU.

- A net read from model_text(name) is the built-in net: the same initial parameters bit for bit (same seed), and after
  three train steps in bf16 and in fp32 the same parameters, gradients and loss bit for bit.
- A file's own initialisation: init_bias and a Gaussian rule on the device, equal to the host's generator
  (model_initial_weights) and within the rule's statistics; one train step stays finite.
"""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MODELS = {"lenet+ref-optimizer": 32, "alexnet+bn": 16, "lcnet": 16, "tiny+logistic+soft-targets": 16}


@pytest.fixture(scope="module")
def env():
    assert torch.cuda.is_available()
    from convnet_b200 import lib, net
    L = lib.load()
    net.load_host()
    yield lib, L, net
    lib.set_precision("tf32")


@pytest.fixture(autouse=True)
def hygiene(env):
    _, L, _ = env
    prec = L.convnet_b200_get_conv_precision()
    try:
        yield
    finally:
        L.convnet_b200_set_conv_precision(prec)
        L.convnet_b200_bf16_invalidate(None)


def _feed(n, seed=7):
    """N(0, 1) input, and uniform labels or a softmax-distributed target per image, from generator `seed`"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n.input_tensor().copy_(torch.randn(n.input_floats, device="cuda", generator=g))
    t = n.targets_tensor()
    if t is None:
        n.labels_tensor().copy_(torch.randint(0, n.num_classes, (n.batch_size,), device="cuda", generator=g,
                                              dtype=torch.int32))
    else:                                                  # column-major [batch x classes]: element n + batch * j
        t.copy_(torch.rand(n.num_classes, n.batch_size, device="cuda", generator=g).softmax(0).reshape(-1))


def _run(N, model, batch, steps=3):
    n = N.Net(model, batch, seed=11)
    try:
        _feed(n)
        first = n.params_tensor().clone()
        losses = [n.train_step() for _ in range(steps)]
        torch.cuda.synchronize()
        return first.cpu(), n.params_tensor().cpu(), n.grads_tensor().cpu(), losses
    finally:
        n.close()


def _bits(t):
    return t.view(torch.int32)


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
@pytest.mark.parametrize("model", sorted(MODELS))
def test_file_net_trains_like_the_built_in(env, tmp_path, model, mode):
    lib, _, N = env
    path = tmp_path / "net.pbtxt"
    path.write_text(N.model_text(model))
    lib.set_precision(mode)
    a = _run(N, model, MODELS[model])
    b = _run(N, str(path), MODELS[model])
    for name, x, y in zip(("initial params", "params", "grads"), a[:3], b[:3]):
        assert torch.equal(_bits(x), _bits(y)), name
    assert np.array(a[3], np.float32).tobytes() == np.array(b[3], np.float32).tobytes(), (a[3], b[3])
    assert all(math.isfinite(v) for v in a[3])


GAUSSIAN_NET = """name: "gauss" seed: 3
layer { name: "input" num_channels: 8 image_size_y: 12 image_size_x: 12 }
layer { name: "conv" num_channels: 32 activation: RECTIFIED_LINEAR }
layer { name: "pool" num_channels: 32 }
layer { name: "output" num_channels: 10 activation: SOFTMAX }
edge { source: "input" dest: "conv" edge_type: CONVOLUTIONAL kernel_size: 5 padding: 2 shared_bias: true
       init_wt: 2.0 init_bias: 1.0 weight_optimizer { epsilon: 0.01 } bias_optimizer { epsilon: 0.01 } }
edge { source: "conv" dest: "pool" edge_type: MAXPOOL kernel_size: 3 stride: 2 }
edge { source: "pool" dest: "output" edge_type: FC initialization: DENSE_GAUSSIAN init_wt: 0.01 init_bias: 1.0
       weight_optimizer { epsilon: 0.01 } bias_optimizer { epsilon: 0.01 } }
"""


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_file_initialisation_on_the_device(env, tmp_path, mode):
    lib, _, N = env
    path = str(tmp_path / "gauss.pbtxt")
    open(path, "w").write(GAUSSIAN_NET)
    lib.set_precision(mode)
    n = N.Net(path, 16, seed=5)
    try:
        p = n.params_tensor().cpu()
        # conv: 32 x (5 x 5 x 8) weights ~ N(0, (2 / sqrt(200))^2), then 32 biases; fc: 10 x (5 x 5 x 32) ~ N(0, 0.01^2)
        for e, (cout, cols, std) in enumerate(((32, 200, 2 / math.sqrt(200)), (10, 800, 0.01))):
            off = n.edges()[[0, 2][e]][2]
            w, b = p[off:off + cout * cols], p[off + cout * cols:off + cout * cols + cout]
            host = torch.tensor(N.model_initial_weights(path, [0, 2][e], seed=5 + 17 * [0, 2][e]))
            assert torch.equal(_bits(w), _bits(host))
            assert torch.equal(b, torch.ones(cout))
            # 6400 / 8000 samples: the sample std within 5 % of the rule's (> 3.5 standard errors), the mean within 5 %
            assert abs(w.double().std().item() / std - 1) < 0.05
            assert abs(w.double().mean().item()) < 0.05 * std
        _feed(n)
        loss = n.train_step()
        assert math.isfinite(loss)
        assert torch.isfinite(n.params_tensor()).all() and torch.isfinite(n.grads_tensor()).all()
    finally:
        n.close()
