"""CPU: the C-ABI shared library loads and exports every symbol include/pixray_b200.h declares (no compute calls),
and the product fails loudly -- never falls back -- when there is no CUDA device."""
import ctypes as C
import os
import re

import pytest
import torch

from pixray_b200 import _lib

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "pixray_b200.h")


def declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pxr_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    lib = _lib.load()
    syms = declared_symbols()
    assert len(syms) >= 20
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, f"declared in the header but not exported: {missing}"
    assert sorted(_lib.EXPORTS) == syms, "pixray_b200/_lib.py EXPORTS is out of sync with the header"


def test_struct_sizes_match_header_layout():
    # pxr_config: 3+1+2+7+8+2+2+1 ints, 2x6 ints, float, (pad), u64, int, float, 3 floats, 8 ints
    assert C.sizeof(_lib.ClipCfg) == 24
    assert C.sizeof(_lib.Config) % 8 == 0
    assert _lib.Config.seed.offset % 8 == 0
    assert C.sizeof(_lib.CutParams) == 8 + 4 + 4 + 8 + 8 + 8  # + color_jitter


def test_test_gemm_desc_fields_follow_the_header():
    """ctypes lays TestGemmDesc out by its field list: it must name the header's fields in the header's order."""
    src = re.sub(r"/\*.*?\*/", "", open(HEADER).read(), flags=re.S)
    body = re.search(r"typedef struct \{([^}]*)\} pxr_test_gemm_desc;", src).group(1)
    names = []
    for decl in filter(None, (d.strip() for d in body.split(";"))):
        first, *rest = decl.split(",")
        names += [re.sub(r"^.*[\s*]", "", first.strip())] + [r.strip() for r in rest]
    assert [f[0] for f in _lib.TestGemmDesc._fields_] == names
    assert names[-1] == "k_splits"


def test_version_string():
    lib = _lib.load()
    assert b"sm_90a" in lib.pxr_version()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    from pixray_b200 import engine as E
    with pytest.raises(E.EngineError):
        E.B200Engine(drawer=E.DRAWER_PIXEL, image_hw=(32, 32), grid=(8, 8), cutn=4, clip=[E.CLIP_ARCH["ViT-B/32"]])
    # and the C entry point itself refuses without a device
    lib = _lib.load()
    cfg = _lib.Config()
    h = C.c_void_p()
    rc = lib.pxr_create(C.byref(cfg), C.byref(h))
    assert rc != 0 and b"no CUDA device" in lib.pxr_last_error(None)
