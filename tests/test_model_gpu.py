"""One model handle for the four models on the GPU: a call made for one kind of model is refused on a handle of another
kind, and a forward pass or train step with dropout is refused on the models that have none."""
import ctypes as C

import numpy as np
import pytest

from distributed_sddmm_b200 import driver as D
from distributed_sddmm_b200 import lib
from oracle import hnh_oracle as orc

pytestmark = pytest.mark.gpu
SEED = 0xC0FFEE + 131


@pytest.fixture(scope="module")
def world():
    D.world_init("self")
    yield
    D.world_finalize()


@pytest.fixture(scope="module")
def models(world):
    N = 64
    rows, cols, _ = orc.er_tuples(6, 4, SEED)
    alg = D.Algorithm("15d_fusion1", D.SpmatLocal.from_tuples(N, N, rows, cols, np.ones(len(rows))), 6, 1)
    return alg, {"GAT": D.GAT(alg, [(6, 4, 2)]), "graph transformer": D.GraphTransformer(alg, [(6, 4, 2)]),
                 "GraphSAGE": D.GraphSAGE(alg, [(6, 4)]), "RGCN": D.RGCN(alg, [(6, 4)], num_relations=2)}


def test_model_specific_calls_refuse_other_kinds(models):
    _, nets = models
    L = lib()
    buf = (C.c_double * 64)()
    p = C.addressof(buf)
    r, c = C.c_int64(), C.c_int64()
    for kind, net in nets.items():
        if kind != "GAT":
            for call in (lambda: L.hnhd_gat_weight_shape(net.h, 0, 0, C.byref(r), C.byref(c)),
                         lambda: L.hnhd_gat_set_weight(net.h, 0, 0, p), lambda: L.hnhd_gat_get_weight_grad(net.h, 0, 0, p),
                         lambda: L.hnhd_gat_set_attention(net.h, b"softmax"),
                         lambda: L.hnhd_gat_get_attention_vectors(net.h, 0, 0, p, p)):
                assert call() == -1 and b"takes a GAT model" in L.hnh_last_error_string(), kind
        if kind != "graph transformer":
            assert L.hnhd_gt_set_edge_attributes(net.h, p, 0, p, 0) == -1
            assert b"takes a graph transformer model" in L.hnh_last_error_string(), kind
    # GAT has no parameters by name
    assert L.hnhd_model_param_shape(nets["GAT"].h, 0, b"weight", C.byref(r), C.byref(c)) == -1
    assert b"(layer, head)" in L.hnh_last_error_string()


@pytest.mark.parametrize("kind", ["GAT", "GraphSAGE", "RGCN"])
def test_dropout_is_refused_without_dropout(models, kind):
    alg, nets = models
    net, L = nets[kind], lib()
    net.set_input(np.ones(net.buffer_shape(0)))
    for dropout in (0.5, float("nan")):
        assert L.hnhd_model_forward(net.h, dropout, 0) == -1 and b"dropout" in L.hnh_last_error_string()
    rows, classes = net.buffer_shape(len(net.layers))
    labels = D.NodeLabels(net, np.zeros(rows, np.int64), classes)
    out = (C.c_double * 4)()
    opt = D.AdamW()
    assert L.hnhd_model_train_step(net.h, labels.h, opt.h, 0.5, 0, out) == -1 and b"dropout" in L.hnh_last_error_string()
    targets = D.LinkTargets(net, alg)
    assert L.hnhd_model_link_train_step(net.h, targets.h, opt.h, 0.5, 0, out) == -1
    assert b"dropout" in L.hnh_last_error_string()
    # refused before any launch: the same model then runs a step without dropout
    assert net.train_step(labels, opt).labelled == rows
