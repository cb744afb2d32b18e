"""Thin Python front end of the C++ host classes (through include/hnh_b200_driver.h).

Mirrors the reference's usage pattern (bench_erdos_renyi.cpp / benchmark_dist.cpp / scratch.cpp):

    world_init()                       # MPI_Init
    S = SpmatLocal.load_er(logM, nnz)  # SpmatLocal S; S.loadTuples(false, logM, nnz, "")
    d_ops = Algorithm("15d_fusion2", S, R, c)   # new Sparse15D_Dense_Shift(&S, R, c, 2, &kernel)
    A, B = d_ops.like_A_matrix(0.001), d_ops.like_B_matrix(0.001)
    Sv, res = d_ops.like_S_values(1.0), d_ops.like_S_values(0.0)
    d_ops.fusedSpMM(A, B, Sv, res, "A")

Everything heavy happens in libhnh_b200.so; numpy arrays cross the boundary only in tests.
"""
from __future__ import annotations

import ctypes as C
import json
import math
import numbers
import os
from typing import NamedTuple

import numpy as np

from ._lib import AlgDims, check, lib

OP = {"sddmmA": 0, "sddmmB": 1, "spmmA": 2, "spmmB": 3, "fusedA": 4, "fusedB": 5, "initial_shift": 6, "de_shift": 7}
KMODE = {"sddmmA": 0, "spmmA": 1, "spmmB": 2, "sddmmB": 3}

_transport_keepalive = None


def world_init(transport: str | None = None):
    """MPI_Init of this library.  transport: None -> from the environment (WORLD_SIZE == 1: self;
    otherwise NCCL on GPU boxes, the gloo-backed External transport on CPU-only boxes)."""
    global _transport_keepalive
    L = lib()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    if transport is None:
        if world == 1:
            transport = "self"
        else:
            import torch
            transport = "nccl" if torch.cuda.is_available() else "gloo"
    if transport == "self":
        check(L.hnhd_init_self(), "hnhd_init_self")
    elif transport == "nccl":
        import torch
        import torch.distributed as dist
        if not dist.is_initialized():
            dist.init_process_group("gloo")
        uid = C.create_string_buffer(128)
        if rank == 0:
            check(L.hnhd_nccl_unique_id(uid), "hnhd_nccl_unique_id")
        t = torch.frombuffer(bytearray(uid.raw), dtype=torch.uint8).clone()
        dist.broadcast(t, src=0)
        check(L.hnhd_init_nccl(rank, world, bytes(t.numpy().tobytes())), "hnhd_init_nccl")
    elif transport == "gloo":
        from .gloo_transport import GlooTransport
        _transport_keepalive = GlooTransport()
        check(L.hnhd_init_external(rank, world, C.byref(_transport_keepalive.table)), "hnhd_init_external")
    else:
        raise ValueError(transport)
    return L.hnhd_world_rank(), L.hnhd_world_size()


def world_finalize(destroy_process_group: bool = True):
    """MPI_Finalize of this library; also tears the torch.distributed group down cleanly."""
    global _transport_keepalive
    check(lib().hnhd_finalize(), "hnhd_finalize")
    _transport_keepalive = None
    if destroy_process_group:
        try:
            import torch.distributed as dist
            if dist.is_available() and dist.is_initialized():
                dist.barrier()
                dist.destroy_process_group()
        except Exception:  # noqa: BLE001
            pass


class SpmatLocal:
    def __init__(self, handle):
        self.h = handle

    @classmethod
    def load_er(cls, logM: int, nnz_per_row: int, seed: int = 0xC0FFEE):
        h = C.c_void_p()
        check(lib().hnhd_spmat_load_er(logM, nnz_per_row, seed, C.byref(h)), "hnhd_spmat_load_er")
        return cls(h)

    @classmethod
    def load_file(cls, filename: str):
        h = C.c_void_p()
        check(lib().hnhd_spmat_load_file(filename.encode(), C.byref(h)), "hnhd_spmat_load_file")
        return cls(h)

    @classmethod
    def from_tuples(cls, M, N, rows, cols, vals):
        rows = np.ascontiguousarray(rows, np.uint64)
        cols = np.ascontiguousarray(cols, np.uint64)
        vals = np.ascontiguousarray(vals, np.float64)
        h = C.c_void_p()
        check(lib().hnhd_spmat_from_tuples(M, N, rows.ctypes.data, cols.ctypes.data, vals.ctypes.data, len(rows),
                                           C.byref(h)), "hnhd_spmat_from_tuples")
        return cls(h)

    def info(self):
        M, N, nnz, loc = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_int64()
        check(lib().hnhd_spmat_info(self.h, C.byref(M), C.byref(N), C.byref(nnz), C.byref(loc)), "hnhd_spmat_info")
        return {"M": M.value, "N": N.value, "dist_nnz": nnz.value, "local_tuples": loc.value}

    def tuples(self):
        n = self.info()["local_tuples"]
        r, c, v = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.zeros(n, np.float64)
        check(lib().hnhd_spmat_tuples(self.h, r.ctypes.data, c.ctypes.data, v.ctypes.data, n), "hnhd_spmat_tuples")
        return r, c, v

    def __del__(self):
        try:
            lib().hnhd_spmat_destroy(self.h)
        except Exception:
            pass


class Dense:
    def __init__(self, handle):
        self.h = handle

    @classmethod
    def create(cls, rows: int, cols: int, value: float = 0.0):
        """A rows x cols device matrix filled with `value` (e.g. the L of Algorithm.sparse_attention)."""
        h = C.c_void_p()
        check(lib().hnhd_dense_create(rows, cols, value, C.byref(h)), "hnhd_dense_create")
        return cls(h)

    @property
    def shape(self):
        r, c = C.c_int64(), C.c_int64()
        lib().hnhd_dense_shape(self.h, C.byref(r), C.byref(c))
        return r.value, c.value

    def fill(self, v):
        check(lib().hnhd_dense_fill(self.h, v), "hnhd_dense_fill")

    def from_host(self, arr):
        arr = np.ascontiguousarray(arr, np.float64)
        assert arr.shape == self.shape, (arr.shape, self.shape)
        check(lib().hnhd_dense_from_host(self.h, arr.ctypes.data), "hnhd_dense_from_host")

    def to_host(self):
        out = np.empty(self.shape, np.float64)
        check(lib().hnhd_dense_to_host(self.h, out.ctypes.data), "hnhd_dense_to_host")
        return out

    def data_ptr(self):
        return lib().hnhd_dense_data(self.h)

    def __del__(self):
        try:
            lib().hnhd_dense_destroy(self.h)
        except Exception:
            pass


class Vec:
    def __init__(self, handle):
        self.h = handle

    @classmethod
    def create(cls, n: int, value: float = 0.0):
        """A device vector of n doubles filled with `value` (e.g. a per-head bias of heads * len(like_S_values()))."""
        h = C.c_void_p()
        check(lib().hnhd_vec_create(int(n), float(value), C.byref(h)), "hnhd_vec_create")
        return cls(h)

    def __len__(self):
        return int(lib().hnhd_vec_size(self.h))

    def fill(self, v):
        check(lib().hnhd_vec_fill(self.h, v), "hnhd_vec_fill")

    def from_host(self, arr):
        arr = np.ascontiguousarray(arr, np.float64)
        assert len(arr) == len(self)
        check(lib().hnhd_vec_from_host(self.h, arr.ctypes.data), "hnhd_vec_from_host")

    def to_host(self):
        out = np.empty(len(self), np.float64)
        check(lib().hnhd_vec_to_host(self.h, out.ctypes.data), "hnhd_vec_to_host")
        return out

    def __del__(self):
        try:
            lib().hnhd_vec_destroy(self.h)
        except Exception:
            pass


def _value_order(mode: str) -> int:
    if mode not in ("A", "B"):
        raise ValueError(f'mode must be "A" or "B", not {mode!r}')
    return 0 if mode == "A" else 1


class Algorithm:
    """A Distributed_Sparse subclass instance with the library's StandardKernel plugged in."""

    def __init__(self, name: str, S: SpmatLocal, R: int, c: int):
        self.name = name
        self.h = C.c_void_p()
        check(lib().hnhd_alg_create(name.encode(), S.h, R, c, C.byref(self.h)), f"hnhd_alg_create({name})")
        d = AlgDims()
        check(lib().hnhd_alg_dims(self.h, C.byref(d)), "hnhd_alg_dims")
        self.dims = d

    def submatrices(self, which):
        n = self.dims.n_a_submatrices if which == "A" else self.dims.n_b_submatrices
        out = np.zeros(4 * n, np.int32)
        lib().hnhd_alg_submatrices(self.h, 0 if which == "A" else 1, out.ctypes.data, 4 * n)
        return out.reshape(n, 4)

    def _mk_dense(self, which, v):
        h = C.c_void_p()
        check(lib().hnhd_dense_like(self.h, which, v, C.byref(h)), "hnhd_dense_like")
        return Dense(h)

    def like_A_matrix(self, v=0.0):
        return self._mk_dense(0, v)

    def like_B_matrix(self, v=0.0):
        return self._mk_dense(1, v)

    def _mk_vec(self, which, v):
        h = C.c_void_p()
        check(lib().hnhd_vec_like(self.h, which, v, C.byref(h)), "hnhd_vec_like")
        return Vec(h)

    def like_S_values(self, v=0.0):
        return self._mk_vec(0, v)

    def like_ST_values(self, v=0.0):
        return self._mk_vec(1, v)

    def dummyInitialize(self, m: Dense, which: str):
        check(lib().hnhd_dense_dummy_initialize(self.h, m.h, 0 if which == "A" else 1), "dummyInitialize")

    def _op(self, op, A, B, S=None, R=None, aux=0):
        # `is not None`, not truth: a Vec has a length, and a rank whose share of S is empty holds vectors of length 0,
        # which must still reach the collective op (the other ranks wait for this one in the ring)
        h = lambda x: x.h if x is not None else None  # noqa: E731
        check(lib().hnhd_alg_op(self.h, OP[op], h(A), h(B), h(S), h(R), aux), op)

    def sddmmA(self, A, B, S, R):
        self._op("sddmmA", A, B, S, R)

    def sddmmB(self, A, B, S, R):
        self._op("sddmmB", A, B, S, R)

    def spmmA(self, A, B, S):
        self._op("spmmA", A, B, S)

    def spmmB(self, A, B, S):
        self._op("spmmB", A, B, S)

    def fusedSpMM(self, A, B, S, R, mode="A"):
        self._op("fusedA" if mode == "A" else "fusedB", A, B, S, R)

    def fusedSpMM_host(self, A, B, S, R, hostA, hostB, hostOut, mode="A", chunk_rows=0):
        """fusedSpMM with host operands (torch CPU tensors or numpy arrays, float64, contiguous; pinned memory
        makes the copies asynchronous).  chunk_rows: 0 default pipeline, < 0 no pipeline."""
        ptr = lambda t: t.data_ptr() if hasattr(t, "data_ptr") else t.ctypes.data  # noqa: E731
        check(lib().hnhd_alg_fused_host(self.h, A.h, B.h, S.h, R.h, ptr(hostA), ptr(hostB), ptr(hostOut),
                                        0 if mode == "A" else 1, chunk_rows), "hnhd_alg_fused_host")

    def edge_softmax(self, values: Vec, mode: str = "A"):
        """In place, collective: values (like_S_values for mode "A", like_ST_values for "B") become their softmax
        over the stored entries of each row of S, on all ranks (Distributed_Sparse::edgeSoftmax)."""
        check(lib().hnhd_alg_edge_softmax(self.h, values.h, _value_order(mode)), "edge_softmax")

    def edge_softmax_backward(self, alpha: Vec, grad: Vec, mode: str = "A"):
        """In place on grad, collective: grad = dL/d alpha becomes dL/d(scores) = alpha * (grad - t), with t the
        row sums of alpha * grad (Distributed_Sparse::edgeSoftmaxBackward)."""
        check(lib().hnhd_alg_edge_softmax_backward(self.h, alpha.h, grad.h, _value_order(mode)), "edge_softmax_backward")

    def additive_scores(self, s: Vec, t: Vec, out: Vec, mode: str = "A", alpha: float = 0.2, derivative: bool = False):
        """out (a value vector of `mode`) = LeakyReLU(s[row] + t[col]) per stored entry of S, or its derivative; s and
        t are whole node vectors (Distributed_Sparse::additiveScores)."""
        check(lib().hnhd_alg_additive_scores(self.h, s.h, t.h, out.h, _value_order(mode), float(alpha), int(derivative)),
              "additive_scores")

    def edge_sums(self, values: Vec, row_sums: Vec, col_sums: Vec):
        """Collective: the row and column sums of an A-order value vector over all ranks (Distributed_Sparse::edgeSums)."""
        check(lib().hnhd_alg_edge_sums(self.h, values.h, row_sums.h, col_sums.h), "edge_sums")

    def gatv2_scores(self, A: Dense, B: Dense, a: Vec, out: Vec, mode: str = "A", alpha: float = 0.2):
        """Collective: out (a value vector of `mode`) = sum_k a_k LeakyReLU(A[u, k] + B[v, k]) per stored entry (u, v)
        of S, with A and B this rank's A- and B-shaped operands (Distributed_Sparse::gatv2Scores)."""
        check(lib().hnhd_alg_gatv2_scores(self.h, A.h, B.h, a.h, out.h, _value_order(mode), float(alpha)), "gatv2_scores")

    def gatv2_backward(self, A: Dense, B: Dense, a: Vec, grad_A: Vec, grad_B: Vec, dA: Dense, dB: Dense, da: Vec,
                       alpha: float = 0.2):
        """Collective: given dL/d scores in both value orders, dA += the gradient of the A side, dB += that of the B side
        (dA and dB may be the same Dense), and da (resized to len(a)) = dL/da summed over all ranks
        (Distributed_Sparse::gatv2Backward)."""
        check(lib().hnhd_alg_gatv2_backward(self.h, A.h, B.h, a.h, grad_A.h, grad_B.h, dA.h, dB.h, da.h, float(alpha)),
              "gatv2_backward")

    @staticmethod
    def _attention_scale(Q: Dense, heads: int, scale):
        if scale is not None:
            return float(scale)
        r = Q.shape[1]
        if heads < 1 or r % heads:
            raise ValueError(f"heads = {heads} must divide the width {r}")
        return 1.0 / math.sqrt(r // heads)

    @staticmethod
    def _dropout_args(dropout, seed):
        """(dropout, seed) as the C ABI takes them: a probability in [0, 1) and an integer in [0, 2^64)."""
        p = float(dropout)
        if not 0.0 <= p < 1.0:
            raise ValueError(f"dropout = {dropout} must lie in [0, 1)")
        if isinstance(seed, bool) or not isinstance(seed, numbers.Integral) or not 0 <= seed < 1 << 64:
            raise ValueError(f"seed = {seed!r} must be an integer in [0, 2^64)")
        return p, int(seed)

    def sparse_attention(self, Q: Dense, K: Dense, V: Dense, Z: Dense, L: Dense, heads: int = 1, scale=None,
                         dropout: float = 0.0, seed: int = 0, bias: Vec = None, edge: Dense = None):
        """Collective: fused attention over the pattern of S (its values are not read).  Q and Z are A-shaped, K and V
        B-shaped, all r wide; per head h of width d = r / heads, Z_u,h = sum over the stored (u, v) of
        softmax_v(scale <Q_u,h, K_v,h>) V_v,h, and L (Dense.create(localArows, heads)) = the rows' log-sum-exp (-inf,
        and Z = 0, for a row without entries).  scale=None means 1/sqrt(d) (Distributed_Sparse::sparseAttention).

        dropout in [0, 1) drops each attention coefficient with that probability and scales the kept ones by
        1 / (1 - dropout), as torch.nn.functional.dropout(softmax(x)) @ V does; L is still the log-sum-exp of all
        scores.  The mask is a hash of (seed, head, global S-row, global S-column), so it does not depend on the
        algorithm or the number of ranks, and duplicate stored (u, v) share one keep bit.  Every rank must pass the
        same dropout and seed, and sparse_attention_backward must get the ones its forward got.

        bias (a Vec, or None) adds b_uv,h to the score of the stored (u, v) in head h, after the scale:
        x_uv,h = scale <Q_u,h, K_v,h> + b_uv,h.  It is an A-order value vector (like_S_values' order) of length n
        (every head reads it) or heads * n (head h reads [h n, (h + 1) n)), n = len(like_S_values()).  b = -inf
        masks an entry (the attn_mask of torch's scaled_dot_product_attention); a row masked throughout gets Z = 0
        and L = -inf, as a row without entries (edge_softmax gives NaN there).  +inf or NaN are not checked and make
        the row NaN.  Contract, not checked: b is a function of the global S-row and S-column (entry_coordinates
        gives them), so stored duplicates of (u, v) share one bias, and every rank passes its part of the same
        bias.  A bias of zeros gives the bits of the call without bias.

        edge (a Dense, or None) holds edge features added to the keys and the values, as PyG's TransformerConv with
        edge_dim does: x_uv,h = scale <Q_u,h, K_v,h + E_uv,h> (+ b_uv,h) and Z_u,h = sum_v softmax(x)_uv (V_v,h +
        E_uv,h) (with dropout's weights).  It is Dense.create(len(like_S_values()), r): row i belongs to entry i of the
        A-order value vector, filled in the order of entry_coordinates("A"), and head h reads its columns
        [h d, (h + 1) d).  It stays on this rank (no ring carries it).  Contract, not checked: E is a function of the
        global S-row and S-column, so stored duplicates of (u, v) share one row, and every rank passes its part of the
        same E.  E = 0 gives the bits of the call without it."""
        s = self._attention_scale(Q, heads, scale)
        p, sd = self._dropout_args(dropout, seed)
        if edge is not None:
            check(lib().hnhd_alg_sparse_attention_edge(self.h, Q.h, K.h, V.h, Z.h, L.h, int(heads), s, p, sd,
                                                       self._vec_arg(bias, "bias"), self._dense_arg(edge, "edge")),
                  "sparse_attention")
        elif bias is None:
            check(lib().hnhd_alg_sparse_attention_dropout(self.h, Q.h, K.h, V.h, Z.h, L.h, int(heads), s, p, sd),
                  "sparse_attention")
        else:
            check(lib().hnhd_alg_sparse_attention_bias(self.h, Q.h, K.h, V.h, Z.h, L.h, int(heads), s, p, sd,
                                                       self._vec_arg(bias, "bias")),
                  "sparse_attention")

    def sparse_attention_backward(self, Q: Dense, K: Dense, V: Dense, Z: Dense, L: Dense, dZ: Dense, dQ: Dense, dK: Dense,
                                  dV: Dense, heads: int = 1, scale=None, dropout: float = 0.0, seed: int = 0,
                                  bias: Vec = None, bias_B: Vec = None, dbias: Vec = None, dbias_B: Vec = None,
                                  edge: Dense = None, edge_B: Dense = None, dedge: Dense = None):
        """Collective: given dZ = dLoss/dZ and the forward's Z and L, overwrites dQ, dK and dV with the gradients of
        sparse_attention (Distributed_Sparse::sparseAttentionBackward).  dropout and seed must be the ones the forward
        got, and the same on every rank: the backward regenerates the forward's mask from them.

        With a bias, the backward needs it in both value orders: `bias` (the forward's, A order) for the dQ pass and
        `bias_B` (B order, like_ST_values' order, of the same head multiplicity) for the dK, dV pass.  Both must
        hold the same b(u, v) for every stored (u, v); build bias_B from entry_coordinates("B").  dbias / dbias_B
        (optional Vecs, resized to their bias's length) receive dLoss/dbias in each order:
        dx_uv,h = alpha_uv (D w <dZ_u,h, V_v,h> - t_u,h), summed over the heads for a shared bias, in a fixed order
        (repeats are bit-identical); 0 at a masked entry.

        With edge features, the backward needs them in both value orders as well: `edge` (the forward's, A order)
        for the dQ pass and `edge_B` (Dense.create(len(like_ST_values()), r), B order, filled from
        entry_coordinates("B")) for the dK, dV pass, holding the same e(u, v) for every stored (u, v).  dedge (an
        optional Dense, resized to edge's shape and overwritten) receives dLoss/dE in the A order:
        dE_uv,h = scale dx_uv,h Q_u,h + D w alpha_uv,h dZ_u,h, 0 at a masked entry."""
        s = self._attention_scale(Q, heads, scale)
        p, sd = self._dropout_args(dropout, seed)
        if edge is None and edge_B is None:
            if dedge is not None:
                raise ValueError("dedge needs the edge features")
        elif edge is None or edge_B is None:
            raise ValueError("edge features need both value orders: edge (A order) and edge_B (B order)")
        if (bias is None) != (bias_B is None):
            raise ValueError("a bias needs both value orders: bias (A order) and bias_B (B order)")
        if bias is None and (dbias is not None or dbias_B is not None):
            raise ValueError("dbias / dbias_B need their bias")
        if edge is not None:
            check(lib().hnhd_alg_sparse_attention_backward_edge(
                self.h, Q.h, K.h, V.h, Z.h, L.h, dZ.h, dQ.h, dK.h, dV.h, int(heads), s, p, sd, self._vec_arg(bias, "bias"),
                self._vec_arg(bias_B, "bias_B"), self._vec_arg(dbias, "dbias"), self._vec_arg(dbias_B, "dbias_B"),
                self._dense_arg(edge, "edge"), self._dense_arg(edge_B, "edge_B"), self._dense_arg(dedge, "dedge")),
                "sparse_attention_backward")
            return
        if bias is None and bias_B is None:
            check(lib().hnhd_alg_sparse_attention_backward_dropout(self.h, Q.h, K.h, V.h, Z.h, L.h, dZ.h, dQ.h, dK.h, dV.h,
                                                                   int(heads), s, p, sd),
                  "sparse_attention_backward")
            return
        check(lib().hnhd_alg_sparse_attention_backward_bias(
            self.h, Q.h, K.h, V.h, Z.h, L.h, dZ.h, dQ.h, dK.h, dV.h, int(heads), s, p, sd, self._vec_arg(bias, "bias"),
            self._vec_arg(bias_B, "bias_B"), self._vec_arg(dbias, "dbias"), self._vec_arg(dbias_B, "dbias_B")),
            "sparse_attention_backward")

    @staticmethod
    def _dense_arg(m, name):
        if m is None:
            return None
        if not isinstance(m, Dense):
            raise TypeError(f"{name} must be a Dense, not {type(m).__name__}")
        return m.h

    @staticmethod
    def _vec_arg(v, name):
        if v is None:
            return None
        if not isinstance(v, Vec):
            raise TypeError(f"{name} must be a Vec, not {type(v).__name__}")
        return v.h

    def entry_coordinates(self, mode: str = "A"):
        """(rows, cols): int64 numpy arrays with the global S-row and S-column of every entry of this rank's value
        vector of `mode` ("A": like_S_values, "B": like_ST_values), in that vector's order -- what a bias of that
        order is built from (Distributed_Sparse::entryCoordinates)."""
        rows, cols = Vec.create(0), Vec.create(0)
        check(lib().hnhd_alg_entry_coordinates(self.h, _value_order(mode), rows.h, cols.h), "entry_coordinates")
        return rows.to_host().astype(np.int64), cols.to_host().astype(np.int64)

    def link_loss(self, H_A: Dense, H_B: Dense, dH_A: Dense | None = None, dH_B: Dense | None = None,
                  scores: Vec | None = None):
        """Link prediction on this algorithm object's S, the target matrix T (collective; Distributed_Sparse::linkLoss):
        s_uv = <H_A[u], H_B[v]> for every stored (u, v) of T, with H_A A-shaped and H_B B-shaped (one Dense may be both),
        and T's stored values the targets y_uv in [0, 1] (an SDDMM, SpMM or FusedMM on this object overwrites them).
        Returns (loss, correct, count): the mean of F.binary_cross_entropy_with_logits(s, y) over T's entries on all
        ranks, the entries with (s > 0) == (y > 0.5), and the entry count.  dH_A / dH_B (optional, the shapes of H_A /
        H_B) are overwritten with the loss's gradients (one Dense passed as both receives their sum; a gradient may not
        be an H); scores (optional, len(like_S_values())) receives s in the A order (entry_coordinates("A"))."""
        out = (C.c_double * 3)()
        check(lib().hnhd_alg_link_loss(self.h, self._dense_arg(H_A, "H_A"), self._dense_arg(H_B, "H_B"),
                                       self._dense_arg(dH_A, "dH_A"), self._dense_arg(dH_B, "dH_B"),
                                       self._vec_arg(scores, "scores"), out), "link_loss")
        return float(out[0]), int(out[1]), int(out[2])

    def distmult_loss(self, H_A: Dense, H_B: Dense, D: Dense, num_relations: int, target: float, inv_count: float,
                      dH_A: Dense | None = None, dH_B: Dense | None = None, dD: Dense | None = None, scores: Vec | None = None,
                      accumulate: bool = False):
        """Relation-aware link prediction on this algorithm object's S, a target matrix T whose stored values are
        relations in [0, num_relations) (collective; Distributed_Sparse::distmultLoss): s_uv = sum_k H_A[u, k] D[rho, k]
        H_B[v, k] for every stored (u, v) of relation rho -- PyG's DistMult, (z[src] * rel_emb[edge_type] *
        z[dst]).sum(-1) -- with H_A A-shaped, H_B B-shaped (one Dense may be both) and D the num_relations x r relation
        table; an entry whose value is no relation contributes nothing.  Every entry's binary cross-entropy against
        `target` (in [0, 1]) is weighted by inv_count.  Returns (loss sum, correct) of this call over all ranks.  dH_A,
        dH_B, dD (optional) receive the gradients, overwritten or, with accumulate, added to (so a positive and a
        negative call sum into one gradient); scores (optional, len(like_S_values())) receives s in the A order."""
        for name, v in (("num_relations", num_relations),):
            if isinstance(v, bool) or not isinstance(v, numbers.Integral):
                raise ValueError(f"{name} = {v!r} must be an integer")
        for name, v in (("target", target), ("inv_count", inv_count)):
            if isinstance(v, bool) or not isinstance(v, numbers.Real):
                raise ValueError(f"{name} = {v!r} must be a number")
        out = (C.c_double * 2)()
        check(lib().hnhd_alg_distmult_loss(self.h, self._dense_arg(H_A, "H_A"), self._dense_arg(H_B, "H_B"),
                                           self._dense_arg(D, "D"), int(num_relations), float(target), float(inv_count),
                                           self._dense_arg(dH_A, "dH_A"), self._dense_arg(dH_B, "dH_B"),
                                           self._dense_arg(dD, "dD"), self._vec_arg(scores, "scores"), int(bool(accumulate)),
                                           out), "distmult_loss")
        return float(out[0]), int(out[1])

    def max_aggregate(self, X: Dense, Z: Dense, C: Dense):
        """Collective: the SpMM over the (max, .) semiring (Distributed_Sparse::maxAggregate).  X is B-shaped, f wide;
        Z and C (A-shaped, f wide: Dense.create(localArows, f)) are overwritten with Z_u,k = max_v X_v,k over the stored
        entries (u, v) of S on all ranks (duplicates count; S's values are not read) and C_u,k = how many of them
        attain it.  A row without entries gets Z = C = 0: torch's zeros(M, f).scatter_reduce(0, u, X[v], "amax",
        include_self=False), PyG's MaxAggregation.  -0.0 and +0.0 tie; which of the two Z holds is not specified."""
        check(lib().hnhd_alg_max_aggregate(self.h, self._dense_arg(X, "X"), self._dense_arg(Z, "Z"),
                                           self._dense_arg(C, "C")), "max_aggregate")

    def max_aggregate_backward(self, X: Dense, Z: Dense, C: Dense, dZ: Dense, dX: Dense, accumulate: bool = False):
        """Collective: given the forward's Z and C and dZ = dLoss/dZ (A-shaped), dX (X's shape) is overwritten -- or,
        with accumulate, added to -- with dX_v,k = sum_u [X_v,k == Z_u,k] dZ_u,k / C_u,k: tied entries share the
        gradient equally, as torch's autograd of scatter_reduce "amax" (Distributed_Sparse::maxAggregateBackward)."""
        check(lib().hnhd_alg_max_aggregate_backward(self.h, self._dense_arg(X, "X"), self._dense_arg(Z, "Z"),
                                                    self._dense_arg(C, "C"), self._dense_arg(dZ, "dZ"),
                                                    self._dense_arg(dX, "dX"), int(bool(accumulate))),
              "max_aggregate_backward")

    MULTI_STATISTICS = {"moments": 1, "max": 2, "min": 4}

    @classmethod
    def _which(cls, which) -> int:
        """The flags of a collection of statistic names (see multi_aggregate)."""
        names = [which] if isinstance(which, str) else list(which)
        if not names or any(n not in cls.MULTI_STATISTICS for n in names) or len(set(names)) != len(names):
            raise ValueError(f"which = {which!r} must be a non-empty set of {tuple(cls.MULTI_STATISTICS)} without repeats")
        return sum(cls.MULTI_STATISTICS[n] for n in names)

    @classmethod
    def multi_aggregate_width(cls, which, f: int) -> int:
        """The width of multi_aggregate's output for the statistics `which` at input width f."""
        return 2 * len(set([which] if isinstance(which, str) else which)) * int(f)

    def multi_aggregate(self, X: Dense, A: Dense, which=("moments", "max", "min")):
        """Collective: several statistics of each S-row's neighbours in one gather pass (Distributed_Sparse::multiAggregate,
        PNA's aggregation).  which: a non-empty collection of "moments", "max" and "min".  X is B-shaped, f wide; A
        (A-shaped, multi_aggregate_width(which, f) wide) is overwritten with the selected f-wide windows in the fixed order
        [sum_v X_v | sum_v X_v^2 | max_v X_v | #ties of the max | min_v X_v | #ties of the min] over the stored entries
        (u, v) of S on all ranks (duplicates count; S's values are not read), every window 0 on a row without entries."""
        w = self._which(which)
        check(lib().hnhd_alg_multi_aggregate(self.h, self._dense_arg(X, "X"), self._dense_arg(A, "A"), w), "multi_aggregate")

    def multi_aggregate_backward(self, X: Dense, A: Dense, dA: Dense, dX: Dense, which=("moments", "max", "min"),
                                 accumulate: bool = False):
        """Collective: given the forward's A and dA = dLoss/dA (A's layout; its count windows are not read), dX (X's shape)
        is overwritten -- or, with accumulate, added to -- with dX_v = sum_u dA_sum[u] + 2 X_v dA_sq[u] + [X_v == max_u]
        dA_max[u] / C_max[u] + [X_v == min_u] dA_min[u] / C_min[u]: tied entries share the gradient of an extreme
        equally (Distributed_Sparse::multiAggregateBackward)."""
        w = self._which(which)
        check(lib().hnhd_alg_multi_aggregate_backward(self.h, self._dense_arg(X, "X"), self._dense_arg(A, "A"),
                                                      self._dense_arg(dA, "dA"), self._dense_arg(dX, "dX"), w,
                                                      int(bool(accumulate))), "multi_aggregate_backward")

    def edge_relu_aggregate(self, X: Dense, E: Dense, A: Dense):
        """Collective: GINE's aggregation (Distributed_Sparse::edgeReluAggregate).  X is B-shaped, f wide; E holds one
        f-wide row per entry of this rank's A value order (len(like_S_values()) x f, in the order of
        entry_coordinates("A")); A (A-shaped, f wide) is overwritten with A_u = sum_i ReLU(X_v + E_i) over the stored
        entries i = (u, v) of S on all ranks (duplicates count; S's values are not read), 0 on a row without entries."""
        check(lib().hnhd_alg_edge_relu_aggregate(self.h, self._dense_arg(X, "X"), self._dense_arg(E, "E"),
                                                 self._dense_arg(A, "A")), "edge_relu_aggregate")

    def edge_relu_aggregate_backward(self, X: Dense, E_A: Dense, E_B: Dense, dA: Dense, dX: Dense, dE: Dense | None = None,
                                     accumulate: bool = False):
        """Collective: given dA = dLoss/dA (A-shaped), dX (X's shape) is overwritten -- or, with accumulate, added to --
        with dX_v = sum_i [X_v + E_i > 0] dA_u, and dE (optional; resized to E_A's shape) with dE_i = [X_v + E_i > 0]
        dA_u for every entry of the A order (Distributed_Sparse::edgeReluAggregateBackward).  E_A and E_B are the edge
        rows of the A and B value orders (entry_coordinates("A") / ("B")), the same e(u, v) in both.  The mask is strict,
        as torch's relu backward."""
        check(lib().hnhd_alg_edge_relu_aggregate_backward(self.h, self._dense_arg(X, "X"), self._dense_arg(E_A, "E_A"),
                                                          self._dense_arg(E_B, "E_B"), self._dense_arg(dA, "dA"),
                                                          self._dense_arg(dX, "dX"), self._dense_arg(dE, "dE"),
                                                          int(bool(accumulate))), "edge_relu_aggregate_backward")

    def relational_aggregate(self, X: Dense, A: Dense, num_relations: int):
        """Collective: R-GCN's aggregation (Distributed_Sparse::relationalAggregate).  The relation of each stored entry
        (u, v) of S is its stored value (SpmatLocal.from_tuples' vals; an SDDMM, SpMM or FusedMM on this object
        overwrites them), an integer in [0, num_relations).  X is B-shaped, f wide; A (A-shaped, num_relations * f wide:
        Dense.create(localArows, R f)) is overwritten with A[u, rho f + k] = the sum of X[v, k] over the entries (u, v)
        of relation rho on all ranks (duplicates count; 0 where there are none).  An entry whose value is not an integer
        in [0, num_relations) -- negative, too large, fractional, infinite or NaN -- contributes nothing."""
        check(lib().hnhd_alg_relational_aggregate(self.h, self._dense_arg(X, "X"), self._dense_arg(A, "A"),
                                                  int(num_relations)), "relational_aggregate")

    def relational_aggregate_backward(self, dA: Dense, dX: Dense, num_relations: int, accumulate: bool = False):
        """Collective: given dA = dLoss/dA (A-shaped, R f wide), dX (B-shaped, f wide) is overwritten -- or, with
        accumulate, added to -- with dX[v] = the sum of dA[u, rho f : rho f + f] over the stored entries (u, v), rho
        their relation (Distributed_Sparse::relationalAggregateBackward)."""
        check(lib().hnhd_alg_relational_aggregate_backward(self.h, self._dense_arg(dA, "dA"), self._dense_arg(dX, "dX"),
                                                           int(num_relations), int(bool(accumulate))),
              "relational_aggregate_backward")

    @staticmethod
    def _comp_arg(comp):
        """comp as a Dense: a Dense as it is, or an R x B array copied to the device."""
        if isinstance(comp, Dense):
            return comp
        c = np.ascontiguousarray(comp, dtype=np.float64)
        if c.ndim != 2 or c.shape[1] < 1:
            raise ValueError(f"comp must be an R x B matrix with B >= 1, got shape {c.shape}")
        d = Dense.create(c.shape[0], c.shape[1])
        if c.size:
            d.from_host(c)
        return d

    def basis_aggregate(self, X: Dense, H: Dense, comp, num_relations: int, scale: Dense | None = None):
        """Collective: R-GCN's aggregation with basis decomposition (Distributed_Sparse::basisAggregate).  The relation
        rho of each stored entry (u, v) of S is its stored value, as for relational_aggregate.  comp (R x B: a numpy
        array or a Dense) mixes the relations into B bases; scale (optional Dense, A-shaped, num_relations wide) weighs
        each (S-row, relation), e.g. 1 / |N_rho(u)| for the mean; without it every weight is 1.  X is B-shaped, f wide;
        H (A-shaped, B f wide: Dense.create(localArows, B f)) is overwritten with
        H[u, b f + k] = the sum of scale[u, rho] comp[rho, b] X[v, k] over the stored entries (u, v) on all ranks."""
        args = (self._dense_arg(X, "X"), self._dense_arg(H, "H"), self._dense_arg(scale, "scale"))
        c = self._comp_arg(comp)
        check(lib().hnhd_alg_basis_aggregate(self.h, args[0], args[1], c.h, int(num_relations), args[2]), "basis_aggregate")

    def basis_aggregate_backward(self, dH: Dense, X: Dense, dX: Dense, comp, num_relations: int, scale: Dense | None = None,
                                 accumulate: bool = False):
        """Collective: given dH = dLoss/dH (A-shaped, B f wide) and the forward's X, comp and scale, dX (B-shaped, f wide)
        is overwritten -- or, with accumulate, added to -- with dX[v] = the sum of scale[u, rho] sum_b comp[rho, b]
        dH[u, b f : b f + f] over the stored entries (u, v).  Returns dLoss/dcomp as an R x B numpy array, summed over
        all ranks (the same on every rank): dcomp[rho, b] = the sum of scale[u, rho] <dH[u, b f : b f + f], X[v]> over
        the stored entries of relation rho (Distributed_Sparse::basisAggregateBackward)."""
        args = (self._dense_arg(dH, "dH"), self._dense_arg(X, "X"), self._dense_arg(dX, "dX"), self._dense_arg(scale, "scale"))
        c = self._comp_arg(comp)
        dcomp = Dense.create(max(int(num_relations), 0), c.shape[1])
        check(lib().hnhd_alg_basis_aggregate_backward(self.h, args[0], args[1], args[2], c.h, dcomp.h, int(num_relations), args[3],
                                                      int(bool(accumulate))), "basis_aggregate_backward")
        return dcomp.to_host()

    def initial_shift(self, A, B, mode):
        self._op("initial_shift", A, B, aux=KMODE[mode])

    def de_shift(self, A, B, mode):
        self._op("de_shift", A, B, aux=KMODE[mode])

    def info(self):
        buf = C.create_string_buffer(1 << 16)
        n = lib().hnhd_alg_info_json(self.h, buf, len(buf))
        if n < 0:
            check(n, "hnhd_alg_info_json")
        return json.loads(buf.value.decode())

    def perf(self):
        buf = C.create_string_buffer(1 << 16)
        n = lib().hnhd_alg_perf_json(self.h, buf, len(buf))
        if n < 0:
            check(n, "hnhd_alg_perf_json")
        return json.loads(buf.value.decode())

    def reset_timers(self):
        check(lib().hnhd_alg_reset_timers(self.h), "reset_timers")

    def als_residuals(self, steps=1):
        """(residual before, residual after) `steps` rounds of ALS-CG on an artificial ground truth."""
        out = (C.c_double * 2)()
        check(lib().hnhd_als_residuals(self.h, steps, out), "hnhd_als_residuals")
        return out[0], out[1]

    def blocks(self, which="S"):
        """Host copies of the local CSR blocks: list of None | dict(rows, cols, transpose, rowStart, col_idx,
        row_idx, values)."""
        w = 0 if which == "S" else 1
        out = []
        L = lib()
        for b in range(L.hnhd_alg_block_count(self.h, w)):
            rows, cols, nnz = C.c_int64(), C.c_int64(), C.c_int64()
            tr, null = C.c_int(), C.c_int()
            check(L.hnhd_alg_block_meta(self.h, w, b, C.byref(rows), C.byref(cols), C.byref(nnz), C.byref(tr),
                                        C.byref(null)), "block_meta")
            if null.value:
                out.append(None)
                continue
            rs = np.zeros(rows.value + 1, np.int64)
            ci, ri = np.zeros(nnz.value, np.int64), np.zeros(nnz.value, np.int64)
            v = np.zeros(nnz.value, np.float64)
            check(L.hnhd_alg_block_arrays(self.h, w, b, rs.ctypes.data, ci.ctypes.data, ri.ctypes.data, v.ctypes.data),
                  "block_arrays")
            out.append(dict(rows=rows.value, cols=cols.value, transpose=bool(tr.value), rowStart=rs, col_idx=ci,
                            row_idx=ri, values=v))
        return out

    def __del__(self):
        try:
            lib().hnhd_alg_destroy(self.h)
        except Exception:
            pass


def setup_times(reset: bool = False) -> dict:
    """Wall-clock seconds of this process' setup phases so far (hnh::SetupPhase)."""
    buf = C.create_string_buffer(1 << 14)
    n = lib().hnhd_setup_times_json(buf, len(buf), int(reset))
    if n < 0:
        check(n, "hnhd_setup_times_json")
    return json.loads(buf.value.decode())


def timer_start():
    check(lib().hnhd_timer_start(), "timer_start")


def timer_stop() -> float:
    ms = C.c_double()
    check(lib().hnhd_timer_stop(C.byref(ms)), "timer_stop")
    return ms.value


def benchmark_algorithm(S: SpmatLocal, name: str, R: int, c: int, fused=True, app="vanilla", trials=5, warmup=0,
                        output_file: str | None = None):
    buf = C.create_string_buffer(1 << 18)
    n = lib().hnhd_benchmark_algorithm(S.h, name.encode(), output_file.encode() if output_file else None, int(fused), R,
                                       c, app.encode(), trials, warmup, buf, len(buf))
    if n < 0:
        check(n, "hnhd_benchmark_algorithm")
    return json.loads(buf.value.decode())


class _Model:
    """What the four models share: one driver handle (hnhd_model_t) with its buffers, forward and backward passes,
    input gradient and train steps.  _PREFIX names the model in RuntimeError texts ("sage_forward failed ...")."""

    _PREFIX = ""

    def _check(self, rc: int, op: str):
        check(rc, f"{self._PREFIX}_{op}")

    def buffer_shape(self, i: int):
        r, c = C.c_int64(), C.c_int64()
        self._check(lib().hnhd_model_buffer_shape(self.h, int(i), C.byref(r), C.byref(c)), "buffer_shape")
        return r.value, c.value

    def set_input(self, x):
        """Make the activations stale: the next backward pass needs a forward pass first."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        if x.shape != self.buffer_shape(0):
            raise ValueError(f"the input is {self.buffer_shape(0)}, got {x.shape}")
        self._check(lib().hnhd_model_set_input(self.h, x.ctypes.data), "set_input")

    def buffer(self, i: int):
        out = np.empty(self.buffer_shape(i), dtype=np.float64)
        self._check(lib().hnhd_model_get_buffer(self.h, int(i), out.ctypes.data), "get_buffer")
        return out

    def forward(self):
        """Collective."""
        self._forward(0.0, 0)

    def _forward(self, dropout, seed):
        p, sd = Algorithm._dropout_args(dropout, seed)
        self._check(lib().hnhd_model_forward(self.h, p, sd), "forward")

    def backward(self, grad_out):
        """Collective: grad_out = dL/d(network output), this rank's rows.  Needs a forward pass since the parameters or
        the input last changed; the gradients are then read with the model's gradient accessors and input_grad."""
        g = np.ascontiguousarray(grad_out, dtype=np.float64)
        last = len(self.layers)
        if g.shape != self.buffer_shape(last):
            raise ValueError(f"the output gradient is {self.buffer_shape(last)}, got {g.shape}")
        self._check(lib().hnhd_model_backward(self.h, g.ctypes.data), "backward")

    def input_grad(self):
        """dL/d(network input), this rank's rows."""
        out = np.empty(self.buffer_shape(0), dtype=np.float64)
        self._check(lib().hnhd_model_get_input_grad(self.h, out.ctypes.data), "get_input_grad")
        return out

    def train_step(self, labels: "NodeLabels", opt: "AdamW") -> "TrainStep":
        """One collective training step on the device: forward, the mean cross-entropy of the output buffer against
        labels over all ranks, backward, clipping and AdamW (see AdamW).  The forward's activations are stale
        afterwards.  Returns TrainStep(loss, correct, labelled, grad_norm)."""
        return self._train_step(labels, opt, 0.0, 0)

    def _train_step(self, labels, opt, dropout, seed):
        p, sd = Algorithm._dropout_args(dropout, seed)
        out = (C.c_double * 4)()
        self._check(lib().hnhd_model_train_step(self.h, _labels_arg(labels), _adamw_arg(opt), p, sd, out), "train_step")
        return TrainStep._of(out)

    def link_train_step(self, targets: "LinkTargets", opt: "AdamW") -> "TrainStep":
        """One collective link-prediction step on the device: forward, the mean binary cross-entropy of the dot-product
        scores <H_u, H_v> of the output buffer H over the entries of the targets' T, backward, clipping and AdamW.
        Returns TrainStep(loss, correct, labelled = T's entry count, grad_norm)."""
        return self._link_train_step(targets, opt, 0.0, 0)

    def _link_train_step(self, targets, opt, dropout, seed):
        p, sd = Algorithm._dropout_args(dropout, seed)
        out = (C.c_double * 4)()
        self._check(lib().hnhd_model_link_train_step(self.h, _link_targets_arg(targets), _adamw_arg(opt), p, sd, out),
                    "link_train_step")
        return TrainStep._of(out)

    def link_evaluate(self, targets: "LinkTargets"):
        """A forward pass without dropout and the link loss without gradients (collective): (loss, correct, count,
        scores), the scores a numpy array in the order of targets.alg_T.entry_coordinates("A") -- for AUC or Hits@K."""
        t = _link_targets_arg(targets)
        out = (C.c_double * 3)()
        scores = Vec.create(0)
        self._check(lib().hnhd_model_link_evaluate(self.h, t, scores.h, out), "link_evaluate")
        return float(out[0]), int(out[1]), int(out[2]), scores.to_host()

    def relational_link_train_step(self, decoder: "DistMultDecoder", targets: "RelationalLinkTargets",
                                   opt: "AdamW") -> "TrainStep":
        """One collective relational link-prediction step on the device: forward, the mean binary cross-entropy of the
        DistMult scores of the output buffer over the pairs of the targets' T_pos (target 1) and T_neg (target 0),
        backward, clipping and AdamW over the model's parameters and then the decoder's relation table.  Returns
        TrainStep(loss, correct, labelled = the pair count, grad_norm)."""
        return self._relational_link_train_step(decoder, targets, opt, 0.0, 0)

    def _relational_link_train_step(self, decoder, targets, opt, dropout, seed):
        p, sd = Algorithm._dropout_args(dropout, seed)
        out = (C.c_double * 4)()
        self._check(lib().hnhd_model_relational_link_train_step(self.h, _distmult_arg(decoder), _relational_targets_arg(targets),
                                                                _adamw_arg(opt), p, sd, out), "relational_link_train_step")
        return TrainStep._of(out)

    def relational_link_evaluate(self, decoder: "DistMultDecoder", targets: "RelationalLinkTargets"):
        """A forward pass without dropout and the relational link loss without gradients (collective): (loss, correct,
        count, scores_pos, scores_neg), the scores numpy arrays in the orders of targets.alg_pos.entry_coordinates("A")
        and targets.alg_neg.entry_coordinates("A") -- for MRR or Hits@K."""
        d, t = _distmult_arg(decoder), _relational_targets_arg(targets)
        out = (C.c_double * 3)()
        sp, sn = Vec.create(0), Vec.create(0)
        self._check(lib().hnhd_model_relational_link_evaluate(self.h, d, t, sp.h, sn.h, out), "relational_link_evaluate")
        return float(out[0]), int(out[1]), int(out[2]), sp.to_host(), sn.to_host()

    def link_rank(self, ranking: "LinkRanking", queries, decoder: "DistMultDecoder" = None) -> "LinkRanks":
        """Filtered link ranking (collective; include/hnh/link_ranking.hpp): a forward pass without dropout, then the
        rank of each query triple's true tail among every corrupted tail and of its true head among every corrupted
        head, the ranking's known triples filtered out, by the DistMult scores of decoder -- or by dot products with
        decoder=None, which needs a ranking of one relation.  queries = (heads, rels, tails), the same on every rank.
        A rank is ((gt + 1) + (ge + 1)) / 2 over the candidates scoring above / at least the true one.  Returns
        LinkRanks(mrr, tail_ranks, head_ranks), the same on every rank; .hits_at(k) gives Hits@K."""
        if not isinstance(ranking, LinkRanking):
            raise TypeError(f"ranking must be a LinkRanking, not {type(ranking).__name__}")
        h, r, t = _triples(queries, "queries")
        tr, hr = np.empty(len(h), np.float64), np.empty(len(h), np.float64)
        mrr = C.c_double()
        self._check(lib().hnhd_model_link_rank(self.h, ranking.h, _distmult_arg(decoder) if decoder is not None else None,
                                               h.ctypes.data, r.ctypes.data, t.ctypes.data, len(h), tr.ctypes.data,
                                               hr.ctypes.data, C.byref(mrr)), "link_rank")
        return LinkRanks(mrr.value, tr, hr)

    def graph_train_step(self, readout: "GraphReadout", labels: "GraphLabels", opt: "AdamW") -> "TrainStep":
        """One collective graph-classification step on the device: forward, the readout's pool and head, the mean
        cross-entropy over the labelled graphs, backward, clipping and AdamW over the model's parameters and then the
        head's.  Returns TrainStep(loss, correct, labelled = the labelled graphs, grad_norm)."""
        return self._graph_train_step(readout, labels, opt, 0.0, 0)

    def _graph_train_step(self, readout, labels, opt, dropout, seed):
        p, sd = Algorithm._dropout_args(dropout, seed)
        out = (C.c_double * 4)()
        self._check(lib().hnhd_model_graph_train_step(self.h, _readout_arg(readout), _graph_labels_arg(labels), _adamw_arg(opt),
                                                      p, sd, out), "graph_train_step")
        return TrainStep._of(out)

    def graph_evaluate(self, readout: "GraphReadout", labels: "GraphLabels"):
        """A forward pass without dropout, the readout and the loss without gradients (collective): (loss, correct,
        labelled, logits), the logits a num_graphs x C numpy array, the same on every rank -- for accuracy or ROC-AUC."""
        r, lab = _readout_arg(readout), _graph_labels_arg(labels)
        out = (C.c_double * 3)()
        logits = np.empty((readout.num_graphs, readout.num_classes), np.float64)
        self._check(lib().hnhd_model_graph_evaluate(self.h, r, lab, logits.ctypes.data, out), "graph_evaluate")
        return float(out[0]), int(out[1]), int(out[2]), logits

    def __del__(self):
        try:
            lib().hnhd_model_destroy(self.h)
        except Exception:
            pass


class _ModelByName(_Model):
    """A model whose parameters are addressed by layer and name; VECTORS are the names of shape (r,)."""

    VECTORS = ()

    def param_names(self):
        return list(self.PARAMS)

    def param_shape(self, layer: int, name: str):
        r, c = C.c_int64(), C.c_int64()
        self._check(lib().hnhd_model_param_shape(self.h, int(layer), name.encode(), C.byref(r), C.byref(c)), "param_shape")
        return (r.value,) if name in self.VECTORS else (r.value, c.value)

    def set_param(self, layer: int, name: str, value):
        """Make the activations stale: the next backward pass needs a forward pass first."""
        shape = self.param_shape(layer, name)
        v = np.ascontiguousarray(value, dtype=np.float64)
        if v.shape != shape:
            raise ValueError(f"{name} of layer {layer} is {shape}, got {v.shape}")
        self._check(lib().hnhd_model_set_param(self.h, int(layer), name.encode(), v.ctypes.data), "set_param")

    def param(self, layer: int, name: str):
        out = np.empty(self.param_shape(layer, name), dtype=np.float64)
        self._check(lib().hnhd_model_get_param(self.h, int(layer), name.encode(), out.ctypes.data), "get_param")
        return out

    def param_grad(self, layer: int, name: str):
        """dL/d param after a backward pass, summed over all ranks (identical on every rank)."""
        out = np.empty(self.param_shape(layer, name), dtype=np.float64)
        self._check(lib().hnhd_model_get_param_grad(self.h, int(layer), name.encode(), out.ctypes.data), "get_param_grad")
        return out


class GAT(_Model):
    """Multi-head graph attention: forward pass and weight / input gradients (include/hnh/gat.hpp).  layers: [(input_features,
    features_per_head, num_heads), ...].  attention: "leaky" (LeakyReLU of the scores, the reference's formula),
    "softmax" (their softmax over each node's neighbours) or "additive" (the softmax of LeakyReLU(a1 . h_u + a2 . h_v),
    Velickovic et al. 2018; a1 and a2 per head through set_attention_vectors, zero by default).  The algorithm object
    must outlive this one.  "gatv2" is GATv2 attention (Brody, Alon and Yahav 2022, shared weights): the softmax of
    a1 . LeakyReLU(h_u + h_v), with a1 set through set_attention_vectors (a2 is not read).  The last layer keeps its
    ReLU (the reference's formula), so GAT's link scores are >= 0 and it cannot score a pair below 0.5: the graph
    transformer is the model for link prediction."""

    ATTENTIONS = ("leaky", "softmax", "additive", "gatv2")
    _PREFIX = "gat"

    def __init__(self, alg: Algorithm, layers, leaky_relu_alpha: float = 0.2, attention: str = "leaky"):
        if attention not in self.ATTENTIONS:
            raise ValueError(f'attention must be "leaky", "softmax", "additive" or "gatv2", not {attention!r}')
        self.alg = alg
        self.layers = [tuple(int(x) for x in l) for l in layers]
        flat = (C.c_int * (3 * len(self.layers)))(*[x for l in self.layers for x in l])
        self.h = C.c_void_p()
        check(lib().hnhd_gat_create(alg.h, len(self.layers), flat, float(leaky_relu_alpha), C.byref(self.h)), "gat_create")
        self.set_attention(attention)

    def set_attention(self, kind: str):
        """"leaky", "softmax", "additive" or "gatv2"; the next backward pass needs a forward pass first."""
        check(lib().hnhd_gat_set_attention(self.h, kind.encode()), "gat_set_attention")
        self.attention = kind

    def weight_shape(self, layer: int, head: int):
        r, c = C.c_int64(), C.c_int64()
        check(lib().hnhd_gat_weight_shape(self.h, layer, head, C.byref(r), C.byref(c)), "gat_weight_shape")
        return r.value, c.value

    def set_weight(self, layer: int, head: int, w):
        w = np.ascontiguousarray(w, dtype=np.float64)
        shape = self.weight_shape(layer, head)
        if w.shape != shape:
            raise ValueError(f"the weight of layer {layer}, head {head} is {shape}, got {w.shape}")
        check(lib().hnhd_gat_set_weight(self.h, layer, head, w.ctypes.data), "gat_set_weight")

    def weight(self, layer: int, head: int):
        """The weight of (layer, head) as the model holds it (e.g. after train steps)."""
        out = np.empty(self.weight_shape(layer, head), dtype=np.float64)
        check(lib().hnhd_gat_get_weight(self.h, layer, head, out.ctypes.data), "gat_get_weight")
        return out

    def set_attention_vectors(self, layer: int, head: int, a1, a2):
        """The attention vectors of (layer, head), features_per_head long each (additive attention reads both, GATv2
        attention a1 only); the next backward pass needs a forward pass first."""
        fph = self.layers[layer][1]
        a1, a2 = (np.ascontiguousarray(a, dtype=np.float64) for a in (a1, a2))
        if a1.shape != (fph,) or a2.shape != (fph,):
            raise ValueError(f"the attention vectors of layer {layer} are ({fph},), got {a1.shape} and {a2.shape}")
        check(lib().hnhd_gat_set_attention_vectors(self.h, layer, head, a1.ctypes.data, a2.ctypes.data),
              "gat_set_attention_vectors")

    def attention_vectors(self, layer: int, head: int):
        """(a1, a2) of (layer, head) as the model holds them (e.g. after train steps)."""
        fph = self.layers[layer][1]
        a1, a2 = np.empty(fph), np.empty(fph)
        check(lib().hnhd_gat_get_attention_vectors(self.h, layer, head, a1.ctypes.data, a2.ctypes.data),
              "gat_get_attention_vectors")
        return a1, a2

    def attention_grads(self, layer: int, head: int):
        """(dL/d a1, dL/d a2) of (layer, head) after a backward pass, summed over all ranks (zero for the vectors the
        attention kind does not read)."""
        fph = self.layers[layer][1]
        da1, da2 = np.empty(fph), np.empty(fph)
        check(lib().hnhd_gat_get_attention_grads(self.h, layer, head, da1.ctypes.data, da2.ctypes.data),
              "gat_get_attention_grads")
        return da1, da2

    def weight_grad(self, layer: int, head: int):
        """dL/d weight (layer, head), summed over all ranks."""
        out = np.empty(self.weight_shape(layer, head), dtype=np.float64)
        check(lib().hnhd_gat_get_weight_grad(self.h, layer, head, out.ctypes.data), "gat_get_weight_grad")
        return out


def _set_edge_attributes(net, set_fn, attr_A, attr_B):
    """Checks the attributes against net.edge_dim and uploads them through the model's set_fn."""
    if not net.edge_dim:
        raise ValueError("the model has no edge features (edge_dim = 0)")
    a, b = (np.ascontiguousarray(x, dtype=np.float64) for x in (attr_A, attr_B))
    for name, x in (("attr_A", a), ("attr_B", b)):
        if x.ndim != 2 or x.shape[1] != net.edge_dim:
            raise ValueError(f"{name} must be n x {net.edge_dim}, got {x.shape}")
    net._check(set_fn(net.h, a.ctypes.data, a.shape[0], b.ctypes.data, b.shape[0]), "set_edge_attributes")


class GraphTransformer(_ModelByName):
    """A graph transformer on fused sparse attention: layers of PyG's TransformerConv(concat=True, root_weight=True)
    with the heads concatenated, forward and backward (include/hnh/graph_transformer.hpp).  layers: [(input_features,
    features_per_head, num_heads), ...]; every layer but the last ends in a ReLU.  edge_dim > 0 adds edge features
    (per-entry attributes, set with set_edge_attributes, projected by each layer's "edge" weight onto the keys and
    values); beta=True the gated skip connection.  ffn_ratio = k >= 1 makes every layer a post-norm transformer block,
    norm2(h + lin2(relu(lin1(h)))) with h = norm1(the TransformerConv output), LayerNorms of epsilon norm_eps and a
    feed-forward network of hidden width k r, and drops the ReLU between layers.  The algorithm object must outlive this
    one.

    Parameters (zero after construction), by layer and name: "query", "key", "value", "skip" (input_features x r),
    "query_bias", "key_bias", "value_bias", "skip_bias" (r), "edge" (edge_dim x r) and "beta" (3r).  A TransformerConv
    state dict maps onto them as lin_query.weight.T -> "query", lin_query.bias -> "query_bias", ..., lin_edge.weight.T
    -> "edge", lin_beta.weight[0] -> "beta".  With blocks: "norm1", "norm1_bias", "norm2", "norm2_bias" (r; the
    LayerNorm weights start at 1) and "ffn1" ((r + 1) x h: vstack(lin1.weight.T, lin1.bias)), "ffn2" ((h + 1) x r)."""

    PROJECTIONS = ("query", "key", "value", "skip")
    VECTORS = ("query_bias", "key_bias", "value_bias", "skip_bias", "beta", "norm1", "norm1_bias", "norm2", "norm2_bias")
    BLOCK = ("norm1", "norm1_bias", "ffn1", "ffn2", "norm2", "norm2_bias")
    _PREFIX = "gt"

    def __init__(self, alg: Algorithm, layers, edge_dim: int = 0, beta: bool = False, ffn_ratio: int = 0,
                 norm_eps: float = 1e-5):
        self.alg = alg
        self.layers = [tuple(int(x) for x in l) for l in layers]
        if any(len(l) != 3 for l in self.layers):
            raise ValueError("layers are (input_features, features_per_head, num_heads) triples")
        if isinstance(edge_dim, bool) or not isinstance(edge_dim, numbers.Integral) or edge_dim < 0:
            raise ValueError(f"edge_dim = {edge_dim!r} must be a non-negative integer")
        if isinstance(ffn_ratio, bool) or not isinstance(ffn_ratio, numbers.Integral) or ffn_ratio < 0:
            raise ValueError(f"ffn_ratio = {ffn_ratio!r} must be a non-negative integer")
        if isinstance(norm_eps, bool) or not isinstance(norm_eps, numbers.Real) or not (math.isfinite(norm_eps) and norm_eps > 0):
            raise ValueError(f"norm_eps = {norm_eps!r} must be finite and > 0")
        self.edge_dim, self.beta = int(edge_dim), bool(beta)
        self.ffn_ratio, self.norm_eps = int(ffn_ratio), float(norm_eps)
        flat = (C.c_int * (3 * len(self.layers)))(*[x for l in self.layers for x in l])
        self.h = C.c_void_p()
        if self.ffn_ratio:
            check(lib().hnhd_gt_create_block(alg.h, len(self.layers), flat, self.edge_dim, int(self.beta), self.ffn_ratio,
                                             self.norm_eps, C.byref(self.h)), "gt_create_block")
        else:
            check(lib().hnhd_gt_create(alg.h, len(self.layers), flat, self.edge_dim, int(self.beta), C.byref(self.h)),
                  "gt_create")

    def param_names(self):
        names = [n for p in self.PROJECTIONS for n in (p, p + "_bias")]
        names += (["edge"] if self.edge_dim else []) + (["beta"] if self.beta else [])
        return names + (list(self.BLOCK) if getattr(self, "ffn_ratio", 0) else [])

    def set_edge_attributes(self, attr_A, attr_B):
        """The edge attributes of this rank's entries: attr_A (len(like_S_values()) x edge_dim) in the order of
        alg.entry_coordinates("A"), attr_B (len(like_ST_values()) x edge_dim) in that of entry_coordinates("B"), both
        holding the same attribute for every stored (u, v)."""
        _set_edge_attributes(self, lib().hnhd_gt_set_edge_attributes, attr_A, attr_B)

    def forward(self, dropout: float = 0.0, seed: int = 0):
        """Collective.  dropout in [0, 1) is the attention dropout of every layer; layer l draws its masks at seed +
        the heads of the layers before it, so no two (layer, head) pairs share one.  Every rank passes the same
        values.  The backward pass regenerates the masks."""
        self._forward(dropout, seed)

    def train_step(self, labels: "NodeLabels", opt: "AdamW", dropout: float = 0.0, seed: int = 0) -> "TrainStep":
        """One collective training step on the device: forward(dropout, seed), the mean cross-entropy of the output
        buffer against labels over all ranks, backward, clipping and AdamW (see AdamW).  The forward's activations are
        stale afterwards.  Returns TrainStep(loss, correct, labelled, grad_norm)."""
        return self._train_step(labels, opt, dropout, seed)

    def link_train_step(self, targets: "LinkTargets", opt: "AdamW", dropout: float = 0.0, seed: int = 0) -> "TrainStep":
        """One collective link-prediction step on the device: forward(dropout, seed), the mean binary cross-entropy of
        the dot-product scores <H_u, H_v> of the output buffer H over the entries of the targets' T, backward, clipping
        and AdamW.  Returns TrainStep(loss, correct, labelled = T's entry count, grad_norm)."""
        return self._link_train_step(targets, opt, dropout, seed)

    def relational_link_train_step(self, decoder: "DistMultDecoder", targets: "RelationalLinkTargets", opt: "AdamW",
                                   dropout: float = 0.0, seed: int = 0) -> "TrainStep":
        """One collective relational link-prediction step on the device: forward(dropout, seed), the mean binary
        cross-entropy of the DistMult scores over the targets' pairs, backward, clipping and AdamW over the model's
        parameters and then the decoder's.  Returns TrainStep(loss, correct, labelled = the pair count, grad_norm)."""
        return self._relational_link_train_step(decoder, targets, opt, dropout, seed)

    def graph_train_step(self, readout: "GraphReadout", labels: "GraphLabels", opt: "AdamW", dropout: float = 0.0,
                         seed: int = 0) -> "TrainStep":
        """One collective graph-classification step on the device: forward(dropout, seed), the readout's pool and
        head, the mean cross-entropy over the labelled graphs, backward, clipping and AdamW over the model's parameters
        and then the head's.  Returns TrainStep(loss, correct, labelled = the labelled graphs, grad_norm)."""
        return self._graph_train_step(readout, labels, opt, dropout, seed)


class GraphSAGE(_ModelByName):
    """GraphSAGE: layers of PyG's SAGEConv(aggr, root_weight=True, project=False, normalize=False), forward and backward
    (include/hnh/graph_sage.hpp).  layers: [(input_features, output_features), ...]; aggr: "mean", "sum" or "max" over
    the stored entries of each S-row on all ranks (duplicates count; a row without entries aggregates to 0).  Every
    layer but the last ends in a ReLU, so the last layer's output is a valid link-prediction embedding.  The algorithm
    object must outlive this one.

    Parameters (zero after construction), by layer and name: "neigh" (input_features x r), "neigh_bias" (r) and
    "root" (input_features x r).  A SAGEConv state dict maps onto them as lin_l.weight.T -> "neigh", lin_l.bias ->
    "neigh_bias" and lin_r.weight.T -> "root"."""

    AGGREGATIONS = ("mean", "sum", "max")
    PARAMS = ("neigh", "neigh_bias", "root")
    VECTORS = ("neigh_bias",)
    _PREFIX = "sage"

    def __init__(self, alg: Algorithm, layers, aggr: str = "mean"):
        self.alg = alg
        self.layers = [tuple(int(x) for x in l) for l in layers]
        if not self.layers or any(len(l) != 2 for l in self.layers):
            raise ValueError("layers are a non-empty list of (input_features, output_features) pairs")
        if aggr not in self.AGGREGATIONS:
            raise ValueError(f"aggr = {aggr!r} must be one of {self.AGGREGATIONS}")
        self.aggr = aggr
        flat = (C.c_int * (2 * len(self.layers)))(*[x for l in self.layers for x in l])
        self.h = C.c_void_p()
        check(lib().hnhd_sage_create(alg.h, len(self.layers), flat, aggr.encode(), C.byref(self.h)), "sage_create")


class RGCN(_ModelByName):
    """R-GCN: layers of PyG's RGCNConv(in, out, num_relations, num_bases, aggr, root_weight=True, bias=True) without
    block decomposition, forward and backward (include/hnh/rgcn.hpp).  The relation of each stored entry of the
    algorithm's S is its stored value, an integer in [0, num_relations); construction refuses any other value on any
    rank.  layers: [(input_features, output_features), ...]; aggr: "mean" or "sum" over the entries of each (S-row,
    relation) on all ranks (duplicates count; an empty one aggregates to 0).  Every layer but the last ends in a ReLU.
    The forward keeps num_relations * input_features doubles per row per layer, or num_bases * input_features with
    bases.  The algorithm object must outlive this one.

    Parameters (zero after construction), by layer and name: "weight" (num_relations * input_features x r), "bias" (r)
    and "root" (input_features x r).  An RGCNConv state dict maps onto them as weight.reshape(-1, r) -> "weight",
    bias -> "bias" and root -> "root", with no transpose.  With num_bases = B (W_rho = sum_b comp[rho, b] V_b),
    "weight" is B * input_features x r (RGCNConv.weight.reshape(-1, r), the bases) and "comp" (num_relations x B) is
    RGCNConv.comp."""

    AGGREGATIONS = ("mean", "sum")
    PARAMS = ("weight", "bias", "root")
    BASIS_PARAMS = ("weight", "comp", "bias", "root")
    VECTORS = ("bias",)
    _PREFIX = "rgcn"

    def __init__(self, alg: Algorithm, layers, num_relations: int, aggr: str = "mean", num_bases: int | None = None):
        self.alg = alg
        self.layers = [tuple(int(x) for x in l) for l in layers]
        if not self.layers or any(len(l) != 2 for l in self.layers):
            raise ValueError("layers are a non-empty list of (input_features, output_features) pairs")
        if any(a[1] != b[0] for a, b in zip(self.layers, self.layers[1:])):
            raise ValueError(f"the layer widths {self.layers} do not chain")
        if aggr not in self.AGGREGATIONS:
            raise ValueError(f"aggr = {aggr!r} must be one of {self.AGGREGATIONS}")
        if int(num_relations) < 1:
            raise ValueError(f"num_relations = {num_relations} must be positive")
        if num_bases is not None and int(num_bases) < 1:
            raise ValueError(f"num_bases = {num_bases} must be positive (or None for no decomposition)")
        self.aggr, self.num_relations = aggr, int(num_relations)
        self.num_bases = None if num_bases is None else int(num_bases)
        flat = (C.c_int * (2 * len(self.layers)))(*[x for l in self.layers for x in l])
        self.h = C.c_void_p()
        if self.num_bases is None:
            check(lib().hnhd_rgcn_create(alg.h, len(self.layers), flat, self.num_relations, aggr.encode(), C.byref(self.h)),
                  "rgcn_create")
        else:
            check(lib().hnhd_rgcn_create_bases(alg.h, len(self.layers), flat, self.num_relations, self.num_bases, aggr.encode(),
                                               C.byref(self.h)), "rgcn_create_bases")

    def _params(self):
        return self.BASIS_PARAMS if getattr(self, "num_bases", None) else self.PARAMS

    def param_names(self):
        return list(self._params())

    def param_shape(self, layer: int, name: str):
        if name not in self._params():
            raise ValueError(f"no parameter {name!r}: one of {self._params()}")
        return super().param_shape(layer, name)


class GIN(_ModelByName):
    """GIN and GINE: layers of PyG's GINConv(nn, eps, train_eps) or, with edge_dim > 0, GINEConv(nn, eps, train_eps,
    edge_dim), with nn = Sequential(Linear(f, h), ReLU(), Linear(h, r)), forward and backward (include/hnh/gin.hpp).
    layers: [(f, h, r), ...].  GIN sums the neighbours X_v of each S-row over its stored entries on all ranks
    (duplicates count; a row without entries aggregates to 0); GINE sums ReLU(X_v + e_uv) with e = attr lin.weight.T +
    lin.bias on the per-entry attributes set with set_edge_attributes.  Then H = M + (1 + eps) X and the MLP.  Every
    layer but the last ends in a ReLU.  eps starts at `eps` and is trained only with train_eps; otherwise it is a
    constant that no optimizer step, weight decay included, moves (its gradient reads 0).  The algorithm object must
    outlive this one.

    Parameters, by layer and name: "lin1" (f x h), "lin1_bias" (h), "lin2" (h x r), "lin2_bias" (r), with edge features
    "edge" (edge_dim x f) and "edge_bias" (f), and "eps" (1); all zero after construction except eps.  A GINConv /
    GINEConv state dict maps onto them as nn.0.weight.T -> "lin1", nn.0.bias -> "lin1_bias", nn.2.weight.T -> "lin2",
    nn.2.bias -> "lin2_bias", lin.weight.T -> "edge", lin.bias -> "edge_bias" and eps -> "eps"."""

    VECTORS = ("lin1_bias", "lin2_bias", "edge_bias", "eps")
    _PREFIX = "gin"

    def __init__(self, alg: Algorithm, layers, edge_dim: int = 0, eps: float = 0.0, train_eps: bool = False):
        self.alg = alg
        self.layers = [tuple(int(x) for x in l) for l in layers]
        if not self.layers or any(len(l) != 3 for l in self.layers):
            raise ValueError("layers are a non-empty list of (input_features, hidden_features, output_features) triples")
        if any(a[2] != b[0] for a, b in zip(self.layers, self.layers[1:])):
            raise ValueError(f"the layer widths {self.layers} do not chain")
        if isinstance(edge_dim, bool) or not isinstance(edge_dim, numbers.Integral) or edge_dim < 0:
            raise ValueError(f"edge_dim = {edge_dim!r} must be a non-negative integer")
        if isinstance(eps, bool) or not isinstance(eps, numbers.Real) or not math.isfinite(eps):
            raise ValueError(f"eps = {eps!r} must be a finite number")
        self.edge_dim, self.eps, self.train_eps = int(edge_dim), float(eps), bool(train_eps)
        flat = (C.c_int * (3 * len(self.layers)))(*[x for l in self.layers for x in l])
        self.h = C.c_void_p()
        check(lib().hnhd_gin_create(alg.h, len(self.layers), flat, self.edge_dim, self.eps, int(self.train_eps),
                                    C.byref(self.h)), "gin_create")

    def param_names(self):
        names = ["lin1", "lin1_bias", "lin2", "lin2_bias"]
        return names + (["edge", "edge_bias"] if self.edge_dim else []) + ["eps"]

    def set_edge_attributes(self, attr_A, attr_B):
        """The edge attributes of this rank's entries: attr_A (len(like_S_values()) x edge_dim) in the order of
        alg.entry_coordinates("A"), attr_B (len(like_ST_values()) x edge_dim) in that of entry_coordinates("B"), both
        holding the same attribute for every stored (u, v)."""
        _set_edge_attributes(self, lib().hnhd_gin_set_edge_attributes, attr_A, attr_B)


def pna_degree_averages(deg):
    """PyG's PNAConv averages of a degree histogram deg (deg[k] = the number of nodes of in-degree k), in fp64:
    (delta_lin, delta_log) = (sum_k k deg[k], sum_k log(k + 1) deg[k]) / sum_k deg[k].  Raises ValueError for a histogram
    that is not a 1-D array of non-negative integers with a positive sum."""
    h = np.asarray(deg)
    if h.ndim != 1 or h.size == 0:
        raise ValueError(f"deg must be a 1-D degree histogram, got shape {h.shape}")
    h = h.astype(np.float64)
    if not np.all(np.isfinite(h)) or np.any(h < 0) or np.any(h != np.round(h)):
        raise ValueError("deg must hold non-negative integer counts")
    total = h.sum()
    if total <= 0:
        raise ValueError("deg counts no node")
    k = np.arange(h.size, dtype=np.float64)
    return float((k * h).sum() / total), float((np.log(k + 1.0) * h).sum() / total)


class PNA(_ModelByName):
    """PNA: layers of PyG's PNAConv(in, out, aggregators, scalers, deg, towers=1, pre_layers=1, post_layers=1,
    divide_input=False, edge_dim=None, train_norm=False), forward and backward (include/hnh/pna.hpp).  layers:
    [(input_features, output_features), ...]; aggregators: an ordered collection of "mean", "sum", "min", "max", "var"
    and "std" over the stored entries of each S-row on all ranks (duplicates count; a row without entries aggregates
    to 0); scalers: of "identity", "amplification", "attenuation", "linear" and "inverse_linear"; deg: the integer
    in-degree histogram PNAConv takes (needed when a scaler reads the degree averages, which are taken in fp64;
    a histogram that is given is always checked).  Min and max
    split their gradient equally over tied entries.  Every layer but the last ends in a ReLU.  The algorithm object must
    outlive this one.  Construction is collective: a bad argument on any rank is refused on every rank.

    Parameters (zero after construction), by layer and name: "pre" (2 input_features x input_features), "pre_bias",
    "post" ((A S + 1) input_features x r), "post_bias", "lin" (r x r) and "lin_bias".  A PNAConv state dict maps onto
    them as pre_nns.0.0.weight.T -> "pre", pre_nns.0.0.bias -> "pre_bias", post_nns.0.0.weight.T -> "post",
    post_nns.0.0.bias -> "post_bias", lin.weight.T -> "lin" and lin.bias -> "lin_bias"."""

    AGGREGATORS = ("mean", "sum", "min", "max", "var", "std")
    SCALERS = ("identity", "amplification", "attenuation", "linear", "inverse_linear")
    DEGREE_SCALERS = ("amplification", "attenuation", "linear", "inverse_linear")  # the scalers that read deg
    PARAMS = ("pre", "pre_bias", "post", "post_bias", "lin", "lin_bias")
    VECTORS = ("pre_bias", "post_bias", "lin_bias")
    _PREFIX = "pna"

    def __init__(self, alg: Algorithm, layers, aggregators=("mean", "min", "max", "std"),
                 scalers=("identity", "amplification", "attenuation"), deg=None):
        self.alg = alg
        self.layers = [tuple(int(x) for x in l) for l in layers]
        if not self.layers or any(len(l) != 2 for l in self.layers):
            raise ValueError("layers are a non-empty list of (input_features, output_features) pairs")
        self.aggregators = [aggregators] if isinstance(aggregators, str) else [str(a) for a in aggregators]
        self.scalers = [scalers] if isinstance(scalers, str) else [str(s) for s in scalers]
        # A refused histogram reaches the collective constructor as NaN averages, which it refuses on every rank, so
        # that no rank is left waiting in the constructor's collectives.  Without a histogram the averages are 0, which
        # the constructor refuses where a scaler reads them.
        problem = None
        if deg is None:
            lin = log = 0.0
            if any(s in self.DEGREE_SCALERS for s in self.scalers):
                problem = f"deg, the degree histogram, is needed by the scalers {self.scalers}"
        else:
            try:
                lin, log = pna_degree_averages(deg)
            except ValueError as e:
                lin = log = math.nan
                problem = str(e)
        self.avg_deg_lin, self.avg_deg_log = lin, log
        flat = (C.c_int * (2 * len(self.layers)))(*[x for l in self.layers for x in l])
        self.h = C.c_void_p()
        rc = lib().hnhd_pna_create(alg.h, len(self.layers), flat, ",".join(self.aggregators).encode(),
                                   ",".join(self.scalers).encode(), lin, log, C.byref(self.h))
        if rc != 0 and problem is not None:
            raise ValueError(problem)
        check(rc, "pna_create")


class TrainStep(NamedTuple):
    """What a train step reports: the mean loss over the labelled rows of all ranks, how many of them the model's
    argmax gets right, how many there are, and the gradient norm before clipping."""
    loss: float
    correct: int
    labelled: int
    grad_norm: float

    @classmethod
    def _of(cls, out):
        return cls(float(out[0]), int(out[1]), int(out[2]), float(out[3]))


class NodeLabels:
    """The node-classification labels of this rank's rows of a model's output buffer, on the device.  labels: an
    integer array of net.buffer_shape(last)[0] entries, each a class in [0, num_classes) or negative for "ignored"
    (padding rows and unlabelled nodes must be negative).  Collective: a bad label on one rank is refused on every
    rank.  The model's algorithm object must outlive this one."""

    def __init__(self, net, labels, num_classes: int):
        lab = np.asarray(labels)
        if lab.dtype.kind not in "iu" or lab.ndim != 1:
            raise ValueError(f"labels must be a 1-D integer array, got {lab.dtype} of shape {lab.shape}")
        rows = net.buffer_shape(len(net.layers))[0]
        if len(lab) != rows:
            raise ValueError(f"{len(lab)} labels for {rows} output rows")
        if len(lab) and (lab.max() > np.iinfo(np.int32).max or lab.min() < np.iinfo(np.int32).min):
            raise ValueError("labels must fit in int32")
        if isinstance(num_classes, bool) or not isinstance(num_classes, numbers.Integral):
            raise ValueError(f"num_classes = {num_classes!r} must be an integer")
        self.num_classes = int(num_classes)
        self._host = np.ascontiguousarray(lab, np.int32)
        self.h = C.c_void_p()
        check(lib().hnhd_labels_create(net.alg.h, self._host.ctypes.data, len(self._host), self.num_classes,
                                       C.byref(self.h)), "labels_create")

    def __del__(self):
        try:
            lib().hnhd_labels_destroy(self.h)
        except Exception:
            pass


class AdamW:
    """torch.optim.AdamW(lr, betas, eps, weight_decay, amsgrad=False, foreach=False) on the device, with one parameter
    group and torch's defaults; max_grad_norm (None: off) clips as torch.nn.utils.clip_grad_norm_ before every step.
    Weight decay applies to every parameter.  An optimizer belongs to the parameters of the first model it steps; the
    lr property may change between steps (a warm-up or decay schedule)."""

    def __init__(self, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 max_grad_norm=None):
        b1, b2 = (float(b) for b in betas)
        mg = 0.0 if max_grad_norm is None else float(max_grad_norm)
        if max_grad_norm is not None and not mg > 0:
            raise ValueError(f"max_grad_norm = {max_grad_norm!r} must be > 0 (None: no clipping)")
        self._lr = float(lr)
        self.h = C.c_void_p()
        check(lib().hnhd_adamw_create(self._lr, b1, b2, float(eps), float(weight_decay), mg, C.byref(self.h)), "adamw_create")

    @property
    def lr(self) -> float:
        return self._lr

    @lr.setter
    def lr(self, value: float):
        check(lib().hnhd_adamw_set_lr(self.h, float(value)), "adamw_set_lr")
        self._lr = float(value)

    def __del__(self):
        try:
            lib().hnhd_adamw_destroy(self.h)
        except Exception:
            pass


class LinkTargets:
    """The link-prediction targets of a model, on the device: alg_T is an Algorithm over the target matrix T, built
    with the model's algorithm name and c over the same nodes (T is square, M = N = the model's S dimensions), whose
    stored values are the targets y_uv in [0, 1] -- 1 for a positive pair, 0 for a negative one, soft targets allowed;
    duplicates count.  Build T with SpmatLocal.from_tuples (e.g. with fresh negatives every epoch).  Collective: a T of
    another layout, a T that is not square, or a target outside [0, 1] on any rank is refused on every rank.  The
    model's and T's algorithm objects must outlive this one."""

    def __init__(self, net, alg_T: Algorithm):
        if not isinstance(alg_T, Algorithm):
            raise TypeError(f"alg_T must be an Algorithm, not {type(alg_T).__name__}")
        self.net, self.alg_T = net, alg_T
        self.h = C.c_void_p()
        check(lib().hnhd_link_targets_create(net.alg.h, alg_T.h, C.byref(self.h)), "link_targets_create")

    def __del__(self):
        try:
            lib().hnhd_link_targets_destroy(self.h)
        except Exception:
            pass


class DistMultDecoder:
    """The DistMult decoder of relational link prediction on the device (include/hnh/distmult.hpp): one relation table
    "rel", num_relations x r with r the width of net's output, zero after construction -- the rel_emb of PyG's
    examples/rgcn_link_pred.py, which maps onto it with no transpose.  net's algorithm object must outlive this one."""

    PARAMS = ("rel",)

    def __init__(self, net, num_relations: int):
        if isinstance(num_relations, bool) or not isinstance(num_relations, numbers.Integral):
            raise ValueError(f"num_relations = {num_relations!r} must be an integer")
        if num_relations < 1:
            raise ValueError(f"num_relations = {num_relations} must be positive")
        self.net, self.num_relations = net, int(num_relations)
        self.width = net.buffer_shape(len(net.layers))[1]
        self.h = C.c_void_p()
        check(lib().hnhd_distmult_create(net.alg.h, self.num_relations, self.width, C.byref(self.h)), "distmult_create")

    def param_names(self):
        return list(self.PARAMS)

    def param_shape(self, name: str):
        r, c = C.c_int64(), C.c_int64()
        check(lib().hnhd_distmult_param_shape(self.h, name.encode(), C.byref(r), C.byref(c)), "distmult_param_shape")
        return r.value, c.value

    def set_param(self, name: str, value):
        shape = self.param_shape(name)
        v = np.ascontiguousarray(value, dtype=np.float64)
        if v.shape != shape:
            raise ValueError(f"{name} is {shape}, got {v.shape}")
        check(lib().hnhd_distmult_set_param(self.h, name.encode(), v.ctypes.data), "distmult_set_param")

    def param(self, name: str):
        out = np.empty(self.param_shape(name), dtype=np.float64)
        check(lib().hnhd_distmult_get_param(self.h, name.encode(), out.ctypes.data), "distmult_get_param")
        return out

    def param_grad(self, name: str):
        """dL/d param after a relational link train step (identical on every rank)."""
        out = np.empty(self.param_shape(name), dtype=np.float64)
        check(lib().hnhd_distmult_get_param_grad(self.h, name.encode(), out.ctypes.data), "distmult_get_param_grad")
        return out

    def __del__(self):
        try:
            lib().hnhd_distmult_destroy(self.h)
        except Exception:
            pass


class RelationalLinkTargets:
    """The relational link-prediction targets of a model, on the device: alg_pos and alg_neg are Algorithms over the
    target matrices T_pos (target 1) and T_neg (target 0; it may have no entry), each built as LinkTargets' T, whose
    stored values are the pairs' relations, integers in [0, num_relations) -- the edge_type of the example.  Duplicates
    count, each under its own relation.  Fresh negatives every epoch are a new alg_neg and a new RelationalLinkTargets.
    Collective: a T of another layout, a T that is not square, or a value that is no relation on any rank is refused
    on every rank.  The three algorithm objects must outlive this one."""

    def __init__(self, net, alg_pos: Algorithm, alg_neg: Algorithm, num_relations: int):
        for name, a in (("alg_pos", alg_pos), ("alg_neg", alg_neg)):
            if not isinstance(a, Algorithm):
                raise TypeError(f"{name} must be an Algorithm, not {type(a).__name__}")
        if isinstance(num_relations, bool) or not isinstance(num_relations, numbers.Integral):
            raise ValueError(f"num_relations = {num_relations!r} must be an integer")
        self.net, self.alg_pos, self.alg_neg, self.num_relations = net, alg_pos, alg_neg, int(num_relations)
        self.h = C.c_void_p()
        check(lib().hnhd_relational_link_targets_create(net.alg.h, alg_pos.h, alg_neg.h, self.num_relations, C.byref(self.h)),
              "relational_link_targets_create")

    def __del__(self):
        try:
            lib().hnhd_relational_link_targets_destroy(self.h)
        except Exception:
            pass


def _triples(triples, what):
    """(heads, rels, tails) as three equally long contiguous int64 arrays."""
    try:
        h, r, t = (np.ascontiguousarray(np.asarray(x).reshape(-1), dtype=np.int64) for x in triples)
    except (TypeError, ValueError) as e:
        raise ValueError(f"{what} must be (heads, rels, tails): {e}") from None
    if not len(h) == len(r) == len(t):
        raise ValueError(f"{what}: heads, rels and tails have {len(h)}, {len(r)} and {len(t)} entries")
    return h, r, t


class LinkRanking:
    """The filter of filtered link ranking on the device's host side (include/hnh/link_ranking.hpp): the known triples
    filter_triples = (heads, rels, tails) of net's nodes, the example's train + valid + test, indexed once by (head,
    relation) and (tail, relation).  Relations lie in [0, num_relations); dot-product ranking (no decoder) uses one
    relation, 0.  Collective: a node outside [0, M), a relation out of range, a layout without full rows, or triples
    that differ between ranks is refused on every rank.  net's algorithm object must outlive this one."""

    def __init__(self, net, filter_triples, num_relations: int = 1):
        if isinstance(num_relations, bool) or not isinstance(num_relations, numbers.Integral):
            raise ValueError(f"num_relations = {num_relations!r} must be an integer")
        self.net, self.num_relations = net, int(num_relations)
        h, r, t = _triples(filter_triples, "filter_triples")
        self.count = len(h)
        self.h = C.c_void_p()
        check(lib().hnhd_link_ranking_create(net.alg.h, h.ctypes.data, r.ctypes.data, t.ctypes.data, len(h), self.num_relations,
                                             C.byref(self.h)), "link_ranking_create")

    def __del__(self):
        try:
            lib().hnhd_link_ranking_destroy(self.h)
        except Exception:
            pass


class LinkRanks(NamedTuple):
    """What link_rank reports: the MRR over all 2 n_q ranks and the tail and head rank of each query."""
    mrr: float
    tail_ranks: np.ndarray
    head_ranks: np.ndarray

    def hits_at(self, k) -> float:
        """The share of the 2 n_q ranks that are <= k (0 for no query)."""
        n = len(self.tail_ranks) + len(self.head_ranks)
        return float(((self.tail_ranks <= k).sum() + (self.head_ranks <= k).sum()) / n) if n else 0.0


class GraphReadout:
    """The readout of graph-level prediction on the device (include/hnh/graph_readout.hpp): pools the rows of net's
    output into one row per graph and, with num_classes, applies a torch.nn.Linear(r, num_classes) head.  batch: this
    rank's graph id of every output row (net.buffer_shape(last)[0] entries, e.g. a slice of PyG's Batch.batch), in [0,
    num_graphs) or negative for a row in no graph (padding rows must be negative); the ids need not be sorted.  pool:
    "sum" (global_add_pool), "mean" (global_mean_pool; an empty graph pools to 0) or "max" (global_max_pool; 0 for an
    empty graph; ties share the gradient equally, -0.0 and +0.0 tying).  num_classes None: no head, and the output
    width is the class count.  Collective: a bad batch on one rank is refused on every rank.  net must outlive this.

    Parameters of the head (zero after construction), by name: "weight" (r x C, Linear.weight.T) and "bias" (C)."""

    POOLS = ("sum", "mean", "max")
    PARAMS = ("weight", "bias")
    VECTORS = ("bias",)

    def __init__(self, net, batch, num_graphs: int, pool: str = "mean", num_classes: int | None = None):
        b = np.asarray(batch)
        if b.dtype.kind not in "iu" or b.ndim != 1:
            raise ValueError(f"batch must be a 1-D integer array, got {b.dtype} of shape {b.shape}")
        if pool not in self.POOLS:
            raise ValueError(f"pool = {pool!r} must be one of {self.POOLS}")
        for name, v in (("num_graphs", num_graphs), ("num_classes", num_classes)):
            if v is not None and (isinstance(v, bool) or not isinstance(v, numbers.Integral)):
                raise ValueError(f"{name} = {v!r} must be an integer")
        if num_classes is not None and num_classes < 1:
            raise ValueError(f"num_classes = {num_classes} must be positive (None: no head)")
        self.net, self.pool_kind, self.num_graphs = net, pool, int(num_graphs)
        self.head = num_classes is not None
        self.num_classes = int(num_classes) if self.head else net.buffer_shape(len(net.layers))[1]
        self._batch = np.ascontiguousarray(b, np.int64)
        self._H = None
        self.h = C.c_void_p()
        check(lib().hnhd_readout_create(net.h, self._batch.ctypes.data, len(self._batch), self.num_graphs, pool.encode(),
                                        int(num_classes or 0), C.byref(self.h)), "readout_create")

    def pool(self, H: Dense) -> Dense:
        """P = the pool of H (a Dense of the model's output shape) over all ranks: a num_graphs x r Dense.  Collective."""
        if not isinstance(H, Dense):
            raise TypeError(f"H must be a Dense, not {type(H).__name__}")
        P = Dense.create(1, 1)
        check(lib().hnhd_readout_pool(self.h, H.h, P.h), "readout_pool")
        self._H = H
        return P

    def pool_backward(self, dP: Dense) -> Dense:
        """dL/dH for the H of the last pool, given dP = dL/dP (num_graphs x r, the same on every rank)."""
        if not isinstance(dP, Dense):
            raise TypeError(f"dP must be a Dense, not {type(dP).__name__}")
        if self._H is None:
            raise ValueError("pool_backward needs a pool first")
        dH = Dense.create(1, 1)
        check(lib().hnhd_readout_pool_backward(self.h, self._H.h, dP.h, dH.h), "readout_pool_backward")
        return dH

    def param_names(self):
        return list(self.PARAMS) if self.head else []

    def param_shape(self, name: str):
        r, c = C.c_int64(), C.c_int64()
        check(lib().hnhd_readout_param_shape(self.h, name.encode(), C.byref(r), C.byref(c)), "readout_param_shape")
        return (r.value,) if name in self.VECTORS else (r.value, c.value)

    def set_param(self, name: str, value):
        shape = self.param_shape(name)
        v = np.ascontiguousarray(value, dtype=np.float64)
        if v.shape != shape:
            raise ValueError(f"{name} is {shape}, got {v.shape}")
        check(lib().hnhd_readout_set_param(self.h, name.encode(), v.ctypes.data), "readout_set_param")

    def param(self, name: str):
        out = np.empty(self.param_shape(name), dtype=np.float64)
        check(lib().hnhd_readout_get_param(self.h, name.encode(), out.ctypes.data), "readout_get_param")
        return out

    def param_grad(self, name: str):
        """dL/d param after a graph train step (identical on every rank)."""
        out = np.empty(self.param_shape(name), dtype=np.float64)
        check(lib().hnhd_readout_get_param_grad(self.h, name.encode(), out.ctypes.data), "readout_get_param_grad")
        return out

    def __del__(self):
        try:
            lib().hnhd_readout_destroy(self.h)
        except Exception:
            pass


class GraphLabels:
    """The labels of a readout's num_graphs graphs on the device: each a class in [0, num_classes) or negative for
    "ignored" (train / validation / test splits), the same array on every rank.  num_classes is the logits' width.
    Collective: labels of another length, a label >= num_classes, or labels differing between ranks are refused on every
    rank.  The readout must outlive this one."""

    def __init__(self, readout: GraphReadout, labels, num_classes: int):
        if not isinstance(readout, GraphReadout):
            raise TypeError(f"readout must be a GraphReadout, not {type(readout).__name__}")
        lab = np.asarray(labels)
        if lab.dtype.kind not in "iu" or lab.ndim != 1:
            raise ValueError(f"labels must be a 1-D integer array, got {lab.dtype} of shape {lab.shape}")
        if len(lab) and (lab.max() > np.iinfo(np.int32).max or lab.min() < np.iinfo(np.int32).min):
            raise ValueError("labels must fit in int32")
        if isinstance(num_classes, bool) or not isinstance(num_classes, numbers.Integral):
            raise ValueError(f"num_classes = {num_classes!r} must be an integer")
        self.readout, self.num_classes = readout, int(num_classes)
        self._host = np.ascontiguousarray(lab, np.int32)
        self.h = C.c_void_p()
        check(lib().hnhd_graph_labels_create(readout.h, self._host.ctypes.data, len(self._host), self.num_classes,
                                             C.byref(self.h)), "graph_labels_create")

    def __del__(self):
        try:
            lib().hnhd_graph_labels_destroy(self.h)
        except Exception:
            pass


def _readout_arg(readout):
    if not isinstance(readout, GraphReadout):
        raise TypeError(f"readout must be a GraphReadout, not {type(readout).__name__}")
    return readout.h


def _graph_labels_arg(labels):
    if not isinstance(labels, GraphLabels):
        raise TypeError(f"labels must be a GraphLabels, not {type(labels).__name__}")
    return labels.h


def _link_targets_arg(targets):
    if not isinstance(targets, LinkTargets):
        raise TypeError(f"targets must be a LinkTargets, not {type(targets).__name__}")
    return targets.h


def _distmult_arg(decoder):
    if not isinstance(decoder, DistMultDecoder):
        raise TypeError(f"decoder must be a DistMultDecoder, not {type(decoder).__name__}")
    return decoder.h


def _relational_targets_arg(targets):
    if not isinstance(targets, RelationalLinkTargets):
        raise TypeError(f"targets must be a RelationalLinkTargets, not {type(targets).__name__}")
    return targets.h


def _labels_arg(labels):
    if not isinstance(labels, NodeLabels):
        raise TypeError(f"labels must be a NodeLabels, not {type(labels).__name__}")
    return labels.h


def _adamw_arg(opt):
    if not isinstance(opt, AdamW):
        raise TypeError(f"opt must be an AdamW, not {type(opt).__name__}")
    return opt.h


def als_run(alg: Algorithm, Agt, Bgt, A0, B0, steps: int = 1, cg_iters: int = 10):
    """Distributed_ALS on caller inputs (this rank's local shards, numpy float64): ground truth from (Agt, Bgt),
    embeddings (A0, B0), `steps` alternating cg_optimizer rounds.  Returns ((residual before, after), A, B)."""
    mats = [np.ascontiguousarray(m, dtype=np.float64) for m in (Agt, Bgt, A0, B0)]
    res = (C.c_double * 2)()
    outA, outB = np.empty_like(mats[2]), np.empty_like(mats[3])
    check(lib().hnhd_als_run(alg.h, *[m.ctypes.data for m in mats], steps, cg_iters, res, outA.ctypes.data, outB.ctypes.data),
          "hnhd_als_run")
    return (res[0], res[1]), outA, outB
