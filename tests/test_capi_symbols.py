"""No-GPU checks of the drop-in boundary: the library loads, exports every symbol include/shifu_b200.h declares,
and every compute entry point fails loudly (never falls back) when no sm_90 device is present."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "shifu_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(sb_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_all_exported_and_bound(sb):
    declared = _declared_symbols()
    assert len(declared) >= 40
    lib = ctypes.CDLL(sb.capi.LIB_PATH)
    missing = [s for s in declared if not hasattr(lib, s)]
    assert not missing, "declared in the header but not exported: %s" % missing
    unbound = [s for s in declared if s not in sb.capi.PROTOTYPES]
    assert not unbound, "exported but not bound in _capi.PROTOTYPES: %s" % unbound
    extra = [s for s in sb.capi.PROTOTYPES if s not in declared]
    assert not extra, "bound but not declared in the header: %s" % extra


def test_desc_struct_layout_matches_header(sb):
    # sizeof(sb_net_desc) = 2 + 32 + 32 + 2 ints, 6 floats, 2 ints = 76 * 4 bytes
    assert ctypes.sizeof(sb.NetDesc) == (2 + 2 * sb.capi.SB_MAX_HIDDEN + 2 + 6 + 2) * 4
    hdr = open(os.path.join(ROOT, "include", "shifu_b200.h")).read()
    assert "#define SB_MAX_HIDDEN %d" % sb.capi.SB_MAX_HIDDEN in hdr


def test_no_cpu_fallback_without_gpu(sb):
    if sb.capi.device_count() > 0:
        pytest.skip("a GPU is present")
    d = sb.make_desc(8, [4], [2])
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Trainer(d)
    assert e.value.code == sb.capi.SB_ERR_CUDA and "no CPU fallback" in str(e.value)
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Model.create(d, np.zeros(8 * 4 + 4 + 4 + 1, np.float32))
    assert e.value.code == sb.capi.SB_ERR_CUDA
    with pytest.raises(sb.ShifuB200Error):
        sb.capi.debug_gemm_bf16(np.zeros((4, 8), np.float32), np.zeros((4, 8), np.float32))


def test_argument_validation_is_host_side(sb):
    bad = sb.make_desc(0, [4], [2])
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Trainer(bad)
    assert e.value.code == sb.capi.SB_ERR_INVALID
    with pytest.raises(sb.ShifuB200Error) as e:
        sb.Model.load("", "in", "out")
    assert e.value.code == sb.capi.SB_ERR_INVALID and "Model path is null" in str(e.value)
    with pytest.raises(sb.ShifuB200Error) as e:   # cfg_cg = 2 (the removed CTA-pair tile) is not a tile configuration
        sb.capi.debug_gemm_bf16(np.zeros((256, 64), np.float32), np.zeros((128, 64), np.float32), cg=2, bn=128)
    assert e.value.code == sb.capi.SB_ERR_INVALID and "not instantiated" in str(e.value)
