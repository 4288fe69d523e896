"""CPU: the argument checks of sealdec_debug_attention (include/sealdec.h).  Every configuration the model never runs is
SEALFM_EINVAL before any device work; a valid one reaches the device check (SEALFM_ENODEVICE without a GPU) and, on a GPU
host, runs."""
import ctypes as C

import numpy as np
import pytest

EINVAL, ENODEVICE = -1, -4


def base_case(kind, arch=0):
    """a small valid case of each kind; the arrays are kept alive in the returned dict"""
    Q, S, B, heads, T, pos = 2, 40, 3, 2, 8, 5
    d = 64 * heads
    arr = dict(src_mask=np.ones((Q, S), np.int32))
    if kind == 0:
        arr["qkv"] = np.zeros((Q * S, 3 * d), np.float32)
    elif kind == 1:
        arr.update(qkv=np.zeros((Q * B, 3 * d), np.float32), kc=np.zeros((T, Q * B, d), np.float32),
                   vc=np.zeros((T, Q * B, d), np.float32), anc=np.tile(np.arange(Q * B, dtype=np.int32)[:, None], (1, T)))
    else:
        arr.update(q=np.zeros((Q * B, d), np.float32), ckv=np.zeros((Q * S, 2 * d), np.float32))
    if arch == 1:
        arr["rel_bias"] = np.zeros((32, heads), np.float32)
    scal = dict(kind=kind, arch=arch, d=d, heads=heads, Q=Q, S=S, B=B, pos=pos, T=T, num_buckets=32, max_distance=128,
                out_split=3)
    return scal, arr


def call(scal, arr, rows):
    from seal_b200._lib import AttnCase, lib
    c = AttnCase()
    for k, v in scal.items():
        setattr(c, k, v)
    for k, v in arr.items():
        setattr(c, k, v.ctypes.data if v is not None else None)
    d = scal["d"]
    out = np.empty((rows, d), np.float32)
    sp = [np.empty((rows, d), np.uint16) for _ in range(3)]
    ovf = np.zeros(1, np.int32)
    kc = np.empty((scal["T"], scal["Q"] * scal["B"], d), np.float32)
    vc = np.empty_like(kc)
    path = np.zeros(1, np.uint32)
    rc = lib.sealdec_debug_attention(C.byref(c), out.ctypes.data, *[s.ctypes.data for s in sp], ovf.ctypes.data,
                                     kc.ctypes.data, vc.ctypes.data, path.ctypes.data)
    return rc, lib.sealfm_last_error().decode()


def have_gpu():
    import torch
    return torch.cuda.is_available()


@pytest.mark.parametrize("kind,arch", [(0, 0), (0, 1), (1, 0), (1, 1), (2, 0)])
def test_valid_case_reaches_the_device_check(kind, arch):
    scal, arr = base_case(kind, arch)
    rc, msg = call(scal, arr, 80 if kind == 0 else 6)
    assert rc == (0 if have_gpu() else ENODEVICE), (rc, msg)


def _bad_cases():
    def m(kind, arch=0, scal=None, arr=None, rows=6):
        return kind, arch, scal or {}, arr or {}, rows
    anc_bad = np.tile(np.arange(6, dtype=np.int32)[:, None], (1, 8)); anc_bad[4, 2] = 6
    anc_neg = anc_bad.copy(); anc_neg[4, 2] = -1
    zero_row = np.ones((2, 40), np.int32); zero_row[1] = 0
    return {
        "head_width": m(0, scal=dict(d=192, heads=2), rows=80),
        "bart_d_over_1024": m(2, scal=dict(d=64 * 17, heads=17)),
        "t5_d_over_4096": m(1, 1, scal=dict(d=64 * 65, heads=65)),
        "S_over_1024": m(2, scal=dict(S=1025)),
        "S_zero": m(0, scal=dict(S=0), rows=80),
        "T_over_128": m(1, scal=dict(T=129)),
        "pos_past_T": m(1, scal=dict(pos=8)),
        "ancestor_past_rows": m(1, arr=dict(anc=anc_bad)),
        "ancestor_negative": m(1, arr=dict(anc=anc_neg)),
        "query_without_key": m(2, arr=dict(src_mask=zero_row)),
        "encoder_query_without_key": m(0, arr=dict(src_mask=zero_row), rows=80),
        "packed_length_zero": m(2, arr=dict(src_off=np.array([0, 40, 40], np.int32))),
        "packed_length_past_S": m(2, arr=dict(src_off=np.array([0, 41, 60], np.int32))),
        "B_over_32": m(1, scal=dict(B=33)),
        "compact_after_first_step": m(1, scal=dict(compact=1)),
        "t5_split_none": m(0, 1, scal=dict(out_split=0), rows=80),
        "t5_bad_buckets": m(1, 1, scal=dict(num_buckets=2)),
        "split_k_on_grouped_cross": m(2, scal=dict(split_ks=2),
                                      arr=dict(split_part=np.zeros((2, 6, 128), np.float32), split_bias=np.zeros(128, np.float32))),
        "split_k_on_rounds_kernel": m(1, scal=dict(B=1, split_ks=2),
                                      arr=dict(split_part=np.zeros((2, 2, 384), np.float32), split_bias=np.zeros(384, np.float32))),
        "ragged_self_attention": m(1, scal=dict(G=1), arr=dict(grp_query=np.zeros(1, np.int32), grp_start=np.array([0, 3], np.int32))),
        "ragged_query_out_of_range": m(2, scal=dict(G=1), arr=dict(grp_query=np.array([2], np.int32), grp_start=np.array([0, 3], np.int32))),
        "ragged_decreasing": m(2, scal=dict(G=2), arr=dict(grp_query=np.zeros(2, np.int32), grp_start=np.array([0, 3, 2], np.int32))),
        "unknown_kind": m(3),
        "unknown_split": m(2, scal=dict(out_split=4)),
    }


@pytest.mark.parametrize("name", sorted(_bad_cases()))
def test_bad_arguments_rejected_before_device_work(name):
    kind, arch, scal_over, arr_over, rows = _bad_cases()[name]
    scal, arr = base_case(min(kind, 2), arch)
    scal["kind"] = kind
    scal.update(scal_over)
    arr.update(arr_over)
    rc, msg = call(scal, arr, rows)
    assert rc == EINVAL, (name, rc, msg)


def test_null_case_rejected():
    from seal_b200._lib import lib
    out = np.empty(1, np.float32); path = np.zeros(1, np.uint32)
    assert lib.sealdec_debug_attention(None, out.ctypes.data, None, None, None, None, None, None, path.ctypes.data) == EINVAL
