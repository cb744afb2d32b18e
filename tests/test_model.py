"""The entry points every model handle shares (hnhd_model_*) refuse null handles and null arguments, without a GPU."""
import ctypes as C

import pytest

_buf = (C.c_double * 8)()
P = C.addressof(_buf)
_i64 = C.c_int64()
I64 = C.byref(_i64)
NAMES = (b"query", b"beta", b"nope", b"norm1", b"ffn2", b"neigh", b"weight", b"comp", b"root")

# (entry point, arguments with a null model handle)
NULL_MODEL = [
    ("hnhd_model_buffer_shape", (None, 0, I64, I64)),
    ("hnhd_model_set_input", (None, P)),
    ("hnhd_model_get_buffer", (None, 0, P)),
    ("hnhd_model_forward", (None, 0.0, 0)),
    ("hnhd_model_backward", (None, P)),
    ("hnhd_model_get_input_grad", (None, P)),
    *[("hnhd_model_param_shape", (None, 0, n, I64, I64)) for n in NAMES],
    *[("hnhd_model_set_param", (None, 0, n, P)) for n in NAMES],
    *[("hnhd_model_get_param", (None, 0, n, P)) for n in NAMES],
    *[("hnhd_model_get_param_grad", (None, 0, n, P)) for n in NAMES],
]


@pytest.mark.parametrize("name,args", NULL_MODEL, ids=[f"{n}-{i}" for i, (n, _) in enumerate(NULL_MODEL)])
def test_null_model_is_refused(hnh, name, args):
    assert getattr(hnh, name)(*args) == -1
    assert b"null" in hnh.hnh_last_error_string()


# the model, the labels or targets, the optimizer: each null in turn, then a null result
@pytest.mark.parametrize("step", ["hnhd_model_train_step", "hnhd_model_link_train_step"])
def test_steps_refuse_null_arguments(hnh, step):
    res = (C.c_double * 4)()
    fn = getattr(hnh, step)
    for args in ((None, P, P), (P, None, P), (P, P, None)):
        assert fn(*args, 0.0, 0, res) == -1 and b"null" in hnh.hnh_last_error_string()
    assert fn(P, P, P, 0.0, 0, None) == -1 and b"null" in hnh.hnh_last_error_string()


def test_link_evaluate_refuses_null_arguments(hnh):
    res = (C.c_double * 3)()
    assert hnh.hnhd_model_link_evaluate(None, P, None, res) == -1
    assert hnh.hnhd_model_link_evaluate(P, None, None, res) == -1
    assert hnh.hnhd_model_link_evaluate(P, P, None, None) == -1
    assert b"null" in hnh.hnh_last_error_string()


def test_destroying_a_null_model_is_a_no_op(hnh):
    hnh.hnhd_model_destroy(None)
