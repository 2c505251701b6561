"""CPU: the kernels of the deterministic entry points (the _det twins) contain no floating-point or shared-memory atomic, and
the twins answer the workspace-size query without a GPU.

The scan reads the SASS of the built library (cuobjdump -sass, names demangled with cu++filt).  A float atomic on global
memory compiles to RED*/ATOM* with a float type (REDG.E.ADD.F32.FTZ.RN.STRONG.GPU for atomicAdd(float*)); a shared-memory
float atomicAdd to an ATOMS.CAST.SPIN compare-and-swap loop.  The self-check asserts that the same scan flags exactly the
atomic kernels of the default path, so a pattern that stopped matching could not let a DET kernel pass silently."""
import ctypes
import os
import re
import shutil
import subprocess

import pytest

from swapping_autoencoder_pytorch_b200 import _lib

# every kernel of the library that reduces with atomics, and its number of instantiations
ATOMIC_KERNELS = {
    "wgrad_wg_kernel": 1, "wgrad_split_kernel": 1, "conv_gather_kernel": 12, "conv_wgrad_kernel": 8,
    "bias_act_bwd_kernel": 2, "modulate_bwd_kernel": 2, "fir_tma_kernel": 2, "torgb_bwd_kernel": 4,
}
# the conv kernels among them carry a trailing `bool DET` template parameter: the DET = true instantiations serve the twins
DET_KERNELS = {k: ATOMIC_KERNELS[k] for k in ("wgrad_wg_kernel", "wgrad_split_kernel", "conv_gather_kernel", "conv_wgrad_kernel")}
# the bandwidth kernels' twins live in csrc/det.cu under their own names (the reduction kernel with them: det_reduce_kernel)
DET_SEPARATE = {"bias_act_bwd_det_kernel": 2, "modulate_bwd_det_kernel": 2, "torgb_bwd_det_kernel": 4, "det_reduce_kernel": 1}


def _tool(name):
    for d in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
        if d and os.path.exists(os.path.join(d, "bin", name)):
            return os.path.join(d, "bin", name)
    found = shutil.which(name)
    assert found, "%s not found (CUDA toolkit)" % name
    return found


@pytest.fixture(scope="module")
def sass():
    """{demangled kernel name: [instruction, ...]} of libsae_b200.so"""
    if not os.path.exists(_lib.LIB_PATH):
        _lib.build_library()
    text = subprocess.run([_tool("cuobjdump"), "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;", line)
        if m and cur is not None:
            cur.append(m.group(1))
    names = list(funcs)
    out = subprocess.run([_tool("cu++filt")], input="\n".join(names) + "\n", capture_output=True, text=True, check=True).stdout
    demangled = out.splitlines()
    assert len(demangled) == len(names)
    return {d: funcs[n] for n, d in zip(names, demangled)}


def _opcode(ins):
    toks = ins.split()
    if toks and toks[0].startswith("@"):
        toks = toks[1:]
    return toks[0] if toks else ""


def _atomics(instructions):
    """the opcodes that break determinism: float atomics on global / generic memory, any shared-memory atomic"""
    bad = []
    for ins in instructions:
        op = _opcode(ins)
        if op.startswith("ATOMS"):
            bad.append(op)
        elif op.startswith(("RED", "ATOM")) and re.search(r"\.(F16|BF16|F16x2|F32|F64)(\.|$)", op):
            bad.append(op)
    return bad


def _split(name):
    """'void sae::k<(int)4, (bool)1>(float *, ...)' -> ('k', '<(int)4, (bool)1>')"""
    m = re.match(r"^(?:void )?sae::(\w+)(<.*?>)?\(", name)
    return (m.group(1), m.group(2) or "") if m else (name, "")


def _base(name):
    return _split(name)[0]


def _is_det(name):
    return _split(name)[1].endswith(("(bool)1>", "true>"))


def test_det_kernels_have_no_float_or_shared_atomics(sass):
    det = {n: ins for n, ins in sass.items() if _base(n) in DET_KERNELS and _is_det(n)}
    det.update({n: ins for n, ins in sass.items() if _base(n) in DET_SEPARATE})
    assert len(det) == sum(DET_KERNELS.values()) + sum(DET_SEPARATE.values()), sorted(det)
    for n, ins in det.items():
        assert ins, n
        assert not _atomics(ins), "%s contains %s" % (n, sorted(set(_atomics(ins))))


def test_scan_flags_every_atomic_kernel_of_the_default_path(sass):
    flagged = {n: _atomics(ins) for n, ins in sass.items() if _atomics(ins)}
    per_kernel = {}
    for n in flagged:
        assert not _is_det(n), n
        per_kernel[_base(n)] = per_kernel.get(_base(n), 0) + 1
    assert per_kernel == ATOMIC_KERNELS, per_kernel
    ops = {op for v in flagged.values() for op in v}
    assert ops == {"REDG.E.ADD.F32.FTZ.RN.STRONG.GPU", "ATOMS.CAST.SPIN"}, ops
    shared = {_base(n) for n, v in flagged.items() if "ATOMS.CAST.SPIN" in v}
    assert shared == {"bias_act_bwd_kernel", "modulate_bwd_kernel", "fir_tma_kernel"}, shared


# ---------------------------------------------------------------------------------------------------- workspace-size query
P = ctypes.c_void_p(1 << 20)      # never dereferenced: the query validates arguments and plans, nothing else


def _geom(N, H, W, C, K, R, S, stride, pad):
    P_ = (H + 2 * pad - R) // stride + 1
    Q_ = (W + 2 * pad - S) // stride + 1
    return _lib.ConvGeom(N, H, W, C, K, R, S, P_, Q_, stride, pad, pad)


def _cases():
    g = _geom(2, 16, 16, 32, 64, 3, 3, 1, 1)
    gm = _geom(2, 32, 32, 64, 64, 3, 3, 1, 1)
    lin = _geom(4, 1, 1, 512, 512, 1, 1, 1, 0)
    G = ctypes.byref
    taps = (ctypes.c_float * 4)(1, 3, 3, 1)
    return {
        "wgrad_wgmma": ("sae_conv2d_wgrad_det", (P, P, P, G(g), 0)),
        "wgrad_generic": ("sae_conv2d_wgrad_det", (P, P, P, G(g), 1)),
        "wgrad_3xtf32": ("sae_conv2d_wgrad_3xtf32_det", (P, P, P, G(g), 0)),
        "wgrad_3xtf32_generic": ("sae_conv2d_wgrad_3xtf32_det", (P, P, P, G(g), 1)),
        "wgrad_modulated": ("sae_conv2d_wgrad_modulated_det", (P, P, P, P, P, P, G(gm))),
        "wgrad_modulated_3xtf32": ("sae_conv2d_wgrad_modulated_3xtf32_det", (P, P, P, P, P, P, G(gm))),
        "fprop_splitk": ("sae_conv2d_fprop_det", (P, P, P, G(lin), None, 1)),
        "dgrad_splitk": ("sae_conv2d_dgrad_det", (P, P, P, G(lin), None, 1)),
        "fprop_3xtf32_splitk": ("sae_conv2d_fprop_3xtf32_det", (P, P, P, P, G(lin), None, 1)),
        "dgrad_3xtf32_splitk": ("sae_conv2d_dgrad_3xtf32_det", (P, P, P, P, G(lin), None, 1)),
        "bias_act": ("sae_bias_act_backward_det", (P, P, P, P, 4096 * 64, 64, 0.2, 1.4, P, 64, P, 1, None)),
        "fir_act": ("sae_fir_act_backward_det", (P, taps, taps, P, P, P, 2, 16, 16, 32, 4, 4, 2, 1, 2, 1, 0.2, 1.4, 1, None)),
        "modulate": ("sae_modulate_backward_det", (P, P, P, P, P, 2, 256, 64, 1)),
        "torgb": ("sae_torgb_backward_det", (P, P, P, P, P, P, 2, 16, 16, 64, 0.1, 3 * 256, 256, 16, 1, 1)),
    }


def test_every_reducing_entry_point_has_a_det_twin():
    assert len(_lib.DET_ENTRY_POINTS) == 12
    assert {v[0] for v in _cases().values()} == set(_lib.DET_ENTRY_POINTS)


@pytest.mark.parametrize("case", sorted(_cases()))
def test_size_query_and_small_workspace_need_no_gpu(case):
    lib = _lib.load()
    name, args = _cases()[case]
    fn = getattr(lib, name)
    size = ctypes.c_int64(-1)
    assert fn(*args, None, ctypes.byref(size), None) == 0, lib.sae_last_error()
    assert size.value > 0 and size.value % 256 == 0
    again = ctypes.c_int64(-1)
    assert fn(*args, None, ctypes.byref(again), None) == 0 and again.value == size.value      # a pure function of the arguments
    small = ctypes.c_int64(size.value - 1)
    assert fn(*args, P, ctypes.byref(small), None) == -1 and b"workspace" in lib.sae_last_error()
    assert fn(*args, None, None, None) == -1


def test_split_k_workspace_is_one_slab_per_split():
    # M = 4 rows, 512 columns, K = 512: 16 k-blocks of 32 -> 4 splits of [4, 512] floats
    lib = _lib.load()
    name, args = _cases()["fprop_splitk"]
    size = ctypes.c_int64(0)
    assert getattr(lib, name)(*args, None, ctypes.byref(size), None) == 0
    assert size.value == 4 * 4 * 512 * 4


def test_deterministic_switch_parsing():
    from swapping_autoencoder_pytorch_b200 import backend
    assert backend.parse_deterministic(None) is False
    assert backend.parse_deterministic("") is False
    assert backend.parse_deterministic("0") is False
    assert backend.parse_deterministic("1") is True
    for bad in ("2", "yes", "true", "on"):
        with pytest.raises(ValueError):
            backend.parse_deterministic(bad)
