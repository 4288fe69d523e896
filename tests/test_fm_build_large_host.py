"""Host-side pieces of the streamed GPU index builder (sealfm_build_gpu_ex): which builder FMIndex picks, the
no-device refusal and the options struct's layout against include/sealfm.h."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GB = 1 << 30


@pytest.mark.parametrize("n,free_dev,host,switch,expect", [
    (10_000_000, 80 * GB, 512 * GB, "gpu", "gpu"),                  # fits the in-memory builder
    (10_000_000, None, 512 * GB, "gpu", "host"),                   # no GPU
    (10_000_000, 80 * GB, 512 * GB, "host", "host"),               # forced
    (10_000_000, None, 512 * GB, "gpu_large", "gpu_large"),        # forced (fails later without a GPU)
    (10_000_000, 80 * GB, 512 * GB, "gpu_large", "gpu_large"),
    (1_500_000_000, 50 * GB, 512 * GB, "gpu", "gpu_large"),         # 40 B/symbol does not fit, 12 B/symbol does
    (3_200_000_000, 80 * GB, 512 * GB, "gpu", "gpu_large"),         # NQ-sized: beyond 32-bit ranks
    (5_500_000_000, 79 * GB, 512 * GB, "gpu", "host"),              # KILT-sized, 32-bit symbols: (12 + 4) B/symbol
    (5_500_000_000, 79 * GB, 40 * GB, "gpu", "host"),               # the pinned suffix array does not fit the host
    (7_000_000_000, 79 * GB, 512 * GB, "gpu", "host"),              # the ISA does not fit the device
    ((1 << 40), 10 ** 15, 10 ** 16, "gpu", "host"),                 # beyond 2^40 rows
])
def test_builder_choice(n, free_dev, host, switch, expect):
    from seal_b200.cpp_modules.fm_index import _choose_builder
    assert _choose_builder(n, free_dev, host, switch) == expect


def test_builder_choice_uses_the_largest_symbol():
    """The wavelet-tree phase needs (12 + L/8) B per symbol (BWT, its sorted copy, CUB's alternate keys, tree bits):
    a KILT-sized text over BART's vocabulary (L = 16) fits 79 GiB, one over 32-bit symbols does not."""
    from seal_b200.cpp_modules.fm_index import _choose_builder, _large_device_bytes
    assert _large_device_bytes(5_500_000_001, 50_274 + 10) == 14 * 5_500_000_001 + (2 << 30)
    assert _choose_builder(5_500_000_000, 79 * GB, 512 * GB, "gpu", max_symbol=50_284) == "gpu_large"
    assert _choose_builder(5_500_000_000, 70 * GB, 512 * GB, "gpu", max_symbol=50_284) == "host"


def test_streamed_builder_out_of_memory_falls_back_to_host(monkeypatch):
    """When the estimate picked the streamed builder but it reports SEALFM_ENOMEM, the host builder takes over; a
    forced SEALB200_BUILD=gpu_large raises instead."""
    from seal_b200.cpp_modules import fm_index
    from seal_b200._lib import SealB200Error
    calls = []
    monkeypatch.setattr(fm_index, "_builder", lambda n, max_symbol=0: "gpu_large")
    monkeypatch.setattr(fm_index.lib, "sealfm_build_gpu_ex", lambda *a: calls.append(a) or -3)
    text = np.array([3, 1, 2, 3, 1, 2, 7], dtype=np.uint64)
    monkeypatch.delenv("SEALB200_BUILD", raising=False)
    fm = fm_index.FMIndex(); fm.initialize(text)
    assert len(calls) == 1 and fm.size() == len(text) + 1
    monkeypatch.setenv("SEALB200_BUILD", "host")
    ref = fm_index.FMIndex(); ref.initialize(text)
    for w in range(5):
        assert np.array_equal(fm.section(w), ref.section(w))
    monkeypatch.setenv("SEALB200_BUILD", "gpu_large")
    with pytest.raises(SealB200Error):
        fm_index.FMIndex().initialize(text)


def test_builder_choice_reads_device_memory(monkeypatch):
    import torch
    from seal_b200.cpp_modules import fm_index
    monkeypatch.delenv("SEALB200_BUILD", raising=False)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "current_device", lambda: 0)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (80 * GB, 80 * GB))
    assert fm_index._builder(10_000_000) == "gpu"
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda dev=None: (24 * GB, 80 * GB))
    monkeypatch.setattr(os, "sysconf", lambda k: {"SC_AVPHYS_PAGES": 1 << 27, "SC_PAGE_SIZE": 4096}[k])   # 512 GiB
    assert fm_index._builder(1_000_000_000) == "gpu_large"
    monkeypatch.setenv("SEALB200_BUILD", "host")
    assert fm_index._builder(10_000_000) == "host"


def test_build_gpu_ex_without_a_device_is_enodevice():
    from seal_b200._lib import lib
    a = np.arange(1, 100, dtype=np.uint64)
    out = C.c_void_p(12345)
    assert lib.sealfm_build_gpu_ex(a.ctypes.data, len(a), 8, 1 << 20, None, C.byref(out)) == -4
    assert out.value is None
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if not has_gpu:
        out = C.c_void_p(12345)
        assert lib.sealfm_build_gpu_ex(a.ctypes.data, len(a), 8, 0, None, C.byref(out)) == -4
        assert out.value is None


def test_options_and_stats_layout_match_the_header(tmp_path):
    from seal_b200._lib import BuildOpts, BuildStats
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "sealfm.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu\\n", sizeof(sealfm_build_opts_t), offsetof(sealfm_build_opts_t, force_wide),\n'
                   '         sizeof(sealfm_build_stats_t), offsetof(sealfm_build_stats_t, round_s));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert got == [C.sizeof(BuildOpts), BuildOpts.force_wide.offset, C.sizeof(BuildStats), BuildStats.round_s.offset]
