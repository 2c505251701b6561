"""CPU: the kernel precision switch (``CudaKernels.precision``, initialised from ``SAE_PRECISION``) and what it selects."""
import pytest

from swapping_autoencoder_pytorch_b200 import _lib, backend


def test_parse_precision():
    assert backend.parse_precision(None) == "tf32"
    assert backend.parse_precision("") == "tf32"
    assert backend.parse_precision("tf32") == "tf32"
    assert backend.parse_precision("fp32") == "fp32"
    assert backend.parse_precision(" FP32 ") == "fp32"
    for bad in ("fp16", "bf16", "3xtf32", "32", "ieee", "true"):
        with pytest.raises(ValueError):
            backend.parse_precision(bad)


def test_environment_sets_the_default(monkeypatch):
    monkeypatch.delenv("SAE_PRECISION", raising=False)
    assert backend.CudaKernels().precision == "tf32"
    monkeypatch.setenv("SAE_PRECISION", "fp32")
    assert backend.CudaKernels().precision == "fp32"
    monkeypatch.setenv("SAE_PRECISION", "tf32")
    assert backend.CudaKernels().precision == "tf32"
    monkeypatch.setenv("SAE_PRECISION", "half")
    with pytest.raises(ValueError):
        backend.CudaKernels()


def test_fp32_mode_turns_every_rounding_off(monkeypatch):
    monkeypatch.delenv("SAE_PRECISION", raising=False)
    k = backend.CudaKernels()
    assert k._round() == 1 and k._round(False) == 0 and k._epi().round_tf32 == 1
    k.round_tf32 = False
    assert k._round() == 0
    k.round_tf32 = True
    k.precision = "fp32"
    assert k._round() == 0 and k._round(True) == 0 and k._epi().round_tf32 == 0 and k._epi(round_tf32=True).round_tf32 == 0
    with pytest.raises(ValueError):
        k.precision = "fp64"
    assert k.precision == "fp32"


def test_split_entry_points_validate_before_touching_the_gpu():
    import ctypes
    lib = _lib.load()
    g = _lib.ConvGeom(1, 4, 4, 8, 8, 3, 3, 4, 4, 1, 1, 1)
    assert lib.sae_conv2d_fprop_3xtf32(None, None, None, None, ctypes.byref(g), None, 0, None) == -1
    assert lib.sae_conv2d_dgrad_3xtf32(None, None, None, None, ctypes.byref(g), None, 0, None) == -1
    assert lib.sae_conv2d_wgrad_3xtf32(None, None, None, ctypes.byref(g), 0, None) == -1
    assert lib.sae_conv2d_fprop_per_sample_3xtf32(None, None, None, None, ctypes.byref(g), None, None) == -1
    assert lib.sae_conv2d_dgrad_per_sample_3xtf32(None, None, None, None, ctypes.byref(g), None, None) == -1
    assert lib.sae_conv2d_wgrad_modulated_3xtf32(None, None, None, None, None, None, ctypes.byref(g), None) == -1
    assert lib.sae_split_tf32(None, None, None, 16, None) == -1
    assert lib.sae_split_tf32(None, None, None, 0, None) == 0


def test_filter_memo_key_carries_the_precision(emulated_kernels):
    """a filter memoised inside filter_reuse() is rebuilt after a precision change; the emulation has no ``precision``
    attribute and reads as "tf32\""""
    import torch
    from swapping_autoencoder_pytorch_b200.stylegan2_op import conv as C
    w = torch.randn(4, 3, 3, 3)
    built = []
    with C.filter_reuse():
        a = C.memo(w, "t", lambda: built.append(1) or len(built))
        assert C.memo(w, "t", lambda: built.append(1) or len(built)) == a
        k = backend.kernels()
        k.precision = "fp32"
        try:
            b = C.memo(w, "t", lambda: built.append(1) or len(built))
        finally:
            del k.precision
        assert b != a and len(built) == 2
