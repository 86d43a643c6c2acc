"""CPU-only: the epilogue fusion plan ConvNet::PlanFusion fixes when a net is built (host logic, no device memory) — which
activation, derivative, dropout and bias-gradient passes of the neighbouring layers ride in each edge's kernels, and which
layers keep a separate activation or derivative pass.  Fused and unfused results are bit-identical by design, so on the
GPU a dropped fusion shows only as extra launches; these tables pin the decisions themselves.

Each edge is written "<up><down><flags>": up = the CNB_ACT_* code ComputeUp applies after the bias (0 none, 1 ReLU,
2 logistic), down = the code whose derivative ComputeDown applies, flags = d dropout_up, s scale_down, b sums_bias_below,
o offers_bias_grad."""
import pytest

from convnet_b200 import net as N

PLANS = {
    # conv / 1x1 / FC fuse the ReLU with their shared bias and the ReLU' mask; pools fuse the mask and sum the bias gradient
    # of the conv below; rnorm fuses the ReLU; the pooled layers are linear, so the edges reading them fuse no derivative
    "alexnet": "10do 01b 10 11dso 11dso 01b 10 11dso 11dso 11dso 11dso 11dso 11dso 11dso 11dso 01b 10do 11dso 01so",
    # a batch-normalised layer: the edge writes the pre-normalisation input with its bias alone, the BN pass the activation
    "alexnet+bn": "00o 01b 10 01so 01so 01b 10 01so 01so 01so 01so 01so 01so 01so 01so 01b 00o 01so 01so",
    # sigma / sigma' ride where ReLU / ReLU' do in the weighted edges' kernels; rnorm and the pools keep ReLU only
    "alexnet+logistic": "20do 00b 00 22dso 22dso 00b 00 22dso 22dso 22dso 22dso 22dso 22dso 22dso 22dso 00b 20do 22dso 02so",
    # the local edges' bias is per output feature: no pool above sums it
    "lcnet": "10do 01b 10do 01b 10d 11ds 11dso 01so",
    # 3-D: the conv edges fuse neither the activation nor the mask; the pools fuse the mask but sum no bias gradient
    "c3d": "00 01 00 01 00 01 00o",
    "tiny": "10do 01b 10 11dso 11dso 01b 00o",
    "lenet": "10do 01b 10do 01b 00o",
}

# per model: the layers (chain index) that keep a separate activation pass / derivative pass; none where not listed
SEPARATE = {
    "alexnet+logistic": ([3, 7], [1, 5, 15]),     # sigma after the rnorm kernels; sigma' before the pool undos
    "c3d": ([1, 3, 5], []),                       # the ReLU of the 3-D conv layers (their derivative: the pool undos)
}


def render(plan):
    flags = "dsbo"
    return " ".join("%d%d%s" % (e["up_act"], e["down_act"],
                                "".join(f for f, name in zip(flags, N.FUSION_FLAGS) if e[name]))
                    for e in plan["edges"])


@pytest.mark.parametrize("model", sorted(PLANS))
def test_fusion_plan(model):
    plan = N.model_fusion(model)
    assert render(plan) == PLANS[model]
    act, deriv = SEPARATE.get(model, ([], []))
    assert [i for i, l in enumerate(plan["layers"]) if l["activation_pass"]] == act
    assert [i for i, l in enumerate(plan["layers"]) if l["deriv_pass"]] == deriv


def test_fusion_plan_does_not_depend_on_the_batch_or_the_optimizer():
    for model, same in (("alexnet", "alexnet+rmsprop"), ("alexnet", "alexnet+ref-optimizer"), ("lenet", "lenet+gradcheck")):
        assert N.model_fusion(model, batch=128) == N.model_fusion(same)


def test_fusion_plan_refuses_what_the_net_refuses(tmp_path, capfd):
    # c3d with its first conv edge LOCAL (the untied kernels are 2-D only)
    lines = N.model_text("c3d").splitlines(keepends=True)
    line = lines.index("  edge_type: CONVOLUTIONAL\n") + 1
    lines[line - 1] = "  edge_type: LOCAL\n"
    path = tmp_path / "local3d.pbtxt"
    path.write_text("".join(lines))
    with pytest.raises(ValueError):
        N.model_fusion(str(path))
    assert "%s:%d: edge 'input:conv1a': LOCAL" % (path, line) in capfd.readouterr().err
