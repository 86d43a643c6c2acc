"""CPU-only: the LOCAL (locally connected) edge in the host's models — parameter counts of `lcnet`, where `+bn` puts
[gamma | beta] of the layers a local edge writes, the optimizers the models give local edges, and the refusal of LOCAL
on 3-D layers (host logic, no device memory)."""
import pytest

from convnet_b200 import net as N

pad = lambda v: (v + 127) // 128 * 128

# lcnet (its text in models.cc): conv1, pool1, conv2, pool2, local3, local4, fc5, output
LCNET_EDGES = [64 * (5 * 5 * 3 + 1), 0, 128 * (3 * 3 * 64 + 1), 0,
               128 * (1152 * 144 + 144),          # local3: 12 x 12 modules, K = 3*3*128, one bias per output feature
               128 * (1152 * 100 + 100),          # local4: 10 x 10 modules
               1024 * (10 * 10 * 128 + 1), 1000 * (1024 + 1)]


def test_lcnet_parameter_counts():
    assert N.model_edge_params("lcnet") == LCNET_EDGES
    assert sum(LCNET_EDGES) == 50222440
    lay = N.model_param_layout("lcnet")
    assert lay["total"] == sum(pad(v) for v in LCNET_EDGES)
    off = 0
    for i, v in enumerate(LCNET_EDGES):
        assert lay["edge_offsets"][i] == off
        off += pad(v)


def test_lcnet_batchnorm_layout_follows_the_local_edges():
    assert [l["name"] for l in N.model_bn_layers("lcnet+bn")] == ["conv1", "conv2", "local3", "local4", "fc5"]
    lay = N.model_param_layout("lcnet+bn")
    eo, bo = lay["edge_offsets"], lay["bn_offsets"]
    for edge, layer in ((4, 5), (5, 6)):            # local3 writes layer 5, local4 layer 6
        assert bo[layer] == eo[edge] + pad(LCNET_EDGES[edge])
        assert eo[edge + 1] == bo[layer] + pad(2 * 128)
    for base in ("lcnet", "localcheck"):             # no other layer moves
        assert N.model_bn_layers(base) == []


@pytest.mark.parametrize("suffix", ["+adagrad", "+rmsprop", "+gradcheck", "+bn+adagrad"])
def test_lcnet_suffixes(suffix):
    assert N.model_edge_params("lcnet" + suffix) == LCNET_EDGES


def test_local_edges_get_the_model_optimizers():
    for e in (4, 5):
        w, b = N.model_edge_optimizer("lcnet", e), N.model_edge_optimizer("lcnet", e, "bias")
        assert (w["epsilon"], w["final_momentum"], b["epsilon"], b["final_momentum"]) == pytest.approx((0.01, 0.9, 0.01, 0.9))
    assert N.model_edge_optimizer("lcnet+rmsprop", 4)["optimizer_type"] in (3, "RMSPROP_SGD")


def test_local_gradcheck_net_shapes():
    # 8x8x4 -local 3x3 p1-> 8x8x8 -avgpool 2/1-> 7x7x8 -local 3x3 s2 p0-> 3x3x8 -fc-> 5
    assert N.model_edge_params("localcheck") == [8 * (36 * 64 + 64), 0, 8 * (72 * 9 + 9), 5 * (72 + 1)]


def test_local_on_3d_layers_is_refused_at_its_line(tmp_path, capfd):
    # c3d with its first conv edge LOCAL: the net construction refuses it at the line of edge_type
    lines = N.model_text("c3d").splitlines(keepends=True)
    line = lines.index("  edge_type: CONVOLUTIONAL\n") + 1
    lines[line - 1] = "  edge_type: LOCAL\n"
    path = tmp_path / "local3d.pbtxt"
    path.write_text("".join(lines))
    with pytest.raises(ValueError):
        N.model_edge_params(str(path))
    assert "%s:%d: edge 'input:conv1a': LOCAL is not supported on 3-D layers" % (path, line) in capfd.readouterr().err
    with pytest.raises(ValueError):
        N.model_param_layout(str(path))
