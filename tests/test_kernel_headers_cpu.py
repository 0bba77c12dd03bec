"""Static CPU test of the kernel headers under skellysim_b200/csrc: a header that defines a non-template __global__
function is compiled into exactly one translation unit (a second copy of such a kernel is a second kernel, loaded and
attributed on its own), and the symmetric and cross pair kernels are compiled only with their host side in
skb_sym.cu.  Reads the sources only: needs no library and no GPU."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "skellysim_b200", "csrc")


def _source(path):
    """The file without comments and string literals."""
    src = open(path).read()
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', " ", src, flags=re.S)


def _includes(path):
    return re.findall(r'^\s*#\s*include\s+"([^"]+)"', open(path).read(), flags=re.M)


def _reached(unit):
    """Every header under csrc/ that `unit` includes, directly or through other headers."""
    seen, todo = set(), [unit]
    while todo:
        for inc in _includes(todo.pop()):
            path = os.path.normpath(os.path.join(CSRC, inc))
            if os.path.dirname(path) == CSRC and os.path.exists(path) and path not in seen:
                seen.add(path)
                todo.append(path)
    return {os.path.basename(p) for p in seen}


def _non_template_kernels(path):
    """Names of the __global__ functions `path` defines (a body follows) without a template header."""
    src = _source(path)
    names = []
    for m in re.finditer(r"\b__global__\b", src):
        head = src[:m.start()].rstrip()
        # the declaration's own start: after the previous statement, block or preprocessor line
        start = max(head.rfind(";"), head.rfind("}"), head.rfind("{"), head.rfind("\n#"))
        if re.search(r"\btemplate\s*<", head[start + 1:]):
            continue
        rest = src[m.end():]
        depth, end = 0, None
        for i, c in enumerate(rest):
            depth += c == "("
            depth -= c == ")"
            if depth == 0 and c in ";{":
                end = i
                break
        if end is not None and rest[end] == "{":
            names.append(re.findall(r"(\w+)\s*\(", rest[:end])[-1])
    return names


def _units():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def test_kernel_headers_are_compiled_into_one_unit():
    kernels = {os.path.basename(h): _non_template_kernels(h) for h in glob.glob(os.path.join(CSRC, "*.cuh"))}
    # the parser finds kernels, and skips templates and declarations
    assert "sym_reduce_kernel" in kernels["sym_kernels.cuh"] and "pair_sym_kernel" not in kernels["sym_kernels.cuh"]
    assert "reduce_partials_kernel" in kernels["pair_kernels.cuh"]
    assert "dense_stream_kernel" not in kernels["stream_kernels.cuh"]
    reached = {os.path.basename(u): _reached(u) for u in _units()}
    units_of = {h: sorted(u for u, hs in reached.items() if h in hs) for h in kernels}
    bad = {h: units_of[h] for h in sorted(kernels) if kernels[h] and len(units_of[h]) != 1}
    assert not bad, f"headers with non-template kernels compiled into other than one unit: {bad}"
    assert units_of["sym_kernels.cuh"] == ["skb_sym.cu"], units_of["sym_kernels.cuh"]
    assert units_of["cross_kernels.cuh"] == ["skb_sym.cu"], units_of["cross_kernels.cuh"]
