"""CPU-side checks of the boundary: the C-ABI library builds, loads and exports every symbol that
include/stylesinger_b200.h declares (no compute calls: there is no GPU in the build container)."""
import ctypes
import os
import re

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(REPO, "include", "stylesinger_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ssb_[a-z0-9_]+)\s*\(", src)))


def test_library_builds_and_exports_header_symbols():
    from stylesinger_b200 import build
    lib_path = build.build(verbose=False)
    lib = ctypes.CDLL(lib_path)
    names = _declared()
    assert len(names) >= 18
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
    lib.ssb_version.restype = ctypes.c_int
    assert lib.ssb_version() >= 100


def test_binding_lists_every_header_symbol():
    from stylesinger_b200 import _lib
    assert sorted(_lib.EXPORTS) == _declared()


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from stylesinger_b200 import synth
    from stylesinger_b200.engine import AcousticModel
    from stylesinger_b200._lib import SsbError
    with pytest.raises(SsbError):
        AcousticModel({}, None)


def test_product_never_imports_oracle():
    pkg = os.path.join(REPO, "stylesinger_b200")
    for root, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                txt = open(os.path.join(root, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt, f


def test_library_reads_no_environment():
    """Every execution choice of the library is derived from the input or the platform, or set through the C ABI (where
    tests can reach it): no environment variable selects a code path."""
    csrc = os.path.join(REPO, "stylesinger_b200", "csrc")
    for f in sorted(os.listdir(csrc)):
        txt = open(os.path.join(csrc, f)).read()
        assert not re.search(r"\bgetenv\s*\(", txt), f"{f} calls getenv"


def test_front_end_argument_checks_need_no_gpu():
    """Geometry / argument validation of the f3 entry points happens before any CUDA call: same error behaviour on any host."""
    import numpy as np
    from stylesinger_b200 import _lib
    lib, C = _lib.lib, ctypes
    h = C.c_void_p()
    # hidden_size other than 256 is refused (params_model.py: model_hidden_size = 256)
    z = np.zeros(4 * 128 * 128, np.float32)
    tab = (C.c_void_p * 1)(z.ctypes.data)
    assert lib.ssb_lstm_encoder_create(C.byref(h), 40, 128, 1, tab, tab, tab, tab, 0, None, None) != 0 and not h.value
    assert b"hidden_size 256" in lib.ssb_last_error()
    assert lib.ssb_lstm_encoder_create(C.byref(h), 40, 256, 0, tab, tab, tab, tab, 0, None, None) != 0
    assert lib.ssb_lstm_encoder_workspace_bytes(None, 4, 160, 1) == 0
    assert lib.ssb_lstm_encoder_forward(None, None, 1, 160, None, 0, None, None, None, None, 0, None) != 0
    # STFT geometry: odd n_fft, hop not a multiple of 16, n_fft too long for the guard band, n_mels not a multiple of 4
    for args in ((16000, 401, 160, 401, 40), (16000, 400, 100, 400, 40), (16000, 4096, 160, 4096, 40), (16000, 400, 160, 400, 42),
                 (16000, 400, 160, 512, 40)):
        assert lib.ssb_melspec_create_ex(C.byref(h), *args, C.c_float(0), C.c_float(8000), C.c_float(1e-6), 1, 1, 0) != 0 and not h.value
    assert lib.ssb_melspec_num_frames(None, 1000) == 0
