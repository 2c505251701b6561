"""CPU: the bandwidth-kernel path table of ``tests/test_gpu_bandwidth_paths.py`` stays complete.

Parses the four sources for their ``__global__`` kernels and for the template instantiations their launchers create, and
fails when a kernel appears neither in a table row nor in the module's documented ``UNREACHED`` list, or when a row names a
kernel the sources do not launch.  A kernel added later without a row fails here, on a machine without a GPU."""
import os
import re

from tests.test_gpu_bandwidth_paths import ROWS, UNREACHED, expected_kernels, kernel_name

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "swapping_autoencoder_pytorch_b200", "csrc")
SOURCES = ("upfirdn2d.cu", "elementwise.cu", "torgb.cu", "train_ops.cu")
TYPE_NAMES = {"uint32_t": "unsigned int", "int64_t": "long"}      # the demangler's spelling


def _strip_comments(src):
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return re.sub(r"//[^\n]*", "", src)


def _expand_macros(src):
    """substitute the function-like one-parameter macros (the ToRGB launch macros) at their call sites"""
    for name, param, body in re.findall(r"#define\s+(\w+)\((\w+)\)\s+([^\n]*)", src):
        src = re.sub(r"#define\s+%s\(%s\)[^\n]*" % (name, param), "", src)
        src = re.sub(r"\b%s\((\w+)\)" % name, lambda m: re.sub(r"\b%s\b" % param, m.group(1), body), src)
    return src


def _split_args(s):
    return [a.strip() for a in s.split(",")] if s.strip() else []


def _template_functions(src):
    """host launch helpers: name -> (parameter names, defaults, body text)"""
    out = {}
    for m in re.finditer(r"template\s*<([^<>]*)>\s*static\s+\w+\s+(\w+)\s*\(", src):
        params, defaults = [], {}
        for p in _split_args(m.group(1)):
            decl, _, default = p.partition("=")
            pname = decl.split()[-1]
            params.append(pname)
            if default:
                defaults[pname] = default.strip()
        start = src.index("{", m.end())
        depth, i = 0, start
        while True:
            depth += {"{": 1, "}": -1}.get(src[i], 0)
            if depth == 0:
                break
            i += 1
        out[m.group(2)] = (params, defaults, m.start(), src[start:i + 1])
    return out


def _normalise(kernel, args):
    if args is None:
        return kernel_name(kernel)
    return kernel_name("%s<%s>" % (kernel, ", ".join(TYPE_NAMES.get(a, a) for a in args)))


def parse_instantiations(src):
    """(all __global__ kernel names, the set of normalised launched instantiations)"""
    src = _expand_macros(_strip_comments(src))
    kernels = set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)\s*\(", src))
    helpers = _template_functions(src)
    found = set()
    for m in re.finditer(r"\b(\w+)\s*(?:<([^<>]*)>)?\s*<<<", src):
        kernel, targs = m.group(1), m.group(2)
        assert kernel in kernels, kernel
        args = _split_args(targs) if targs is not None else None
        if args is None or all(re.fullmatch(r"-?\d+|uint32_t|int64_t", a) for a in args):
            found.add(_normalise(kernel, args))
            continue
        # a launch inside a template helper: resolve its parameters from every call of the helper
        owner = [(name, h) for name, h in helpers.items() if h[2] < m.start() and m.group(0) in h[3]]
        assert len(owner) >= 1, "cannot resolve the template arguments of %s" % m.group(0)
        name, (params, defaults, _, body) = max(owner, key=lambda o: o[1][2])
        consts = dict(re.findall(r"constexpr\s+int\s+(\w+)\s*=\s*(\d+)\s*;", body))
        calls = re.findall(r"\b%s\s*<([^<>]*)>\s*\(" % name, src)
        assert calls, "no call of %s" % name
        for call in calls:
            values = dict(defaults)
            values.update(zip(params, _split_args(call)))
            values.update(consts)
            found.add(_normalise(kernel, [values.get(a, a) for a in args]))
    return kernels, found


def _all_sources():
    kernels, found = set(), set()
    for f in SOURCES:
        with open(os.path.join(CSRC, f)) as fh:
            k, i = parse_instantiations(fh.read())
        kernels |= k
        found |= i
    return kernels, found


def test_every_kernel_has_a_row_or_a_reason():
    kernels, found = _all_sources()
    # every __global__ kernel is launched somewhere (else it would escape the check below)
    launched = {re.sub(r"<.*", "", f) for f in found}
    assert kernels == launched, sorted(kernels ^ launched)
    covered = set()
    for row in ROWS:
        covered |= expected_kernels(row)
    missing = sorted(found - covered - set(UNREACHED))
    assert not missing, "kernels with neither a row in the path table nor an UNREACHED reason: %s" % missing


def test_rows_name_real_kernels():
    _, found = _all_sources()
    unknown = sorted({k for row in ROWS for k in expected_kernels(row)} - found)
    assert not unknown, "path-table rows expect kernels the sources never launch: %s" % unknown
    assert set(UNREACHED) <= found, sorted(set(UNREACHED) - found)
    assert not set(UNREACHED) & {k for row in ROWS for k in expected_kernels(row)}


def test_row_ids_unique():
    ids = [r[0] for r in ROWS]
    assert len(ids) == len(set(ids))


def test_parser_sees_template_instantiations():
    """the resolver follows template helpers, their default arguments, local constants and launch macros"""
    _, found = _all_sources()
    for k in ("fir_tma_kernel<3,3,0>", "fir_tma_kernel<4,4,2>", "fir_sep_strip_kernel<2,2,16,2>", "fir_sep_up2_kernel<1,1>",
              "fir_strip_kernel<4,4,8>", "torgb_bwd_kernel<8>", "bias_act_kernel<4,unsignedint>", "modulate_kernel<long>",
              "split_tf32_kernel", "adam_advance_kernel"):
        assert k in found, (k, sorted(found))
