"""Static CPU test of the flow modules under skellysim_b200/csrc: a flow evaluates through its own one-device
evaluators (skb::Evaluator) and never through the multi-device evaluator context of include/skelly_b200.h, and the
shared header skb_internal.hpp keeps its types inside namespace skb.  Reads the sources only: needs no library and no
GPU."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "skellysim_b200", "csrc")

FLOW_MODULES = ["skb_flow.cu", "skb_flow.hpp", "skb_matvec.cu", "skb_system.cu", "skb_listener.cu", "skb_solve.cu",
                "skb_step.cu", "skb_mflow.cu"]


def _source(name):
    """The file without comments and string literals."""
    src = open(os.path.join(CSRC, name)).read()
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', " ", src, flags=re.S)


def test_flow_modules_do_not_use_the_context():
    pattern = re.compile(r"\bskb_ctx\b|\bDeviceState\b|\bskb_set_\w+\s*\(|\bskb_ctx_\w+\s*\(|\bdevs\s*\[\s*0\s*\]")
    # the pattern finds what it should
    assert pattern.search("skb_set_targets(c, r, n)") and pattern.search("fl->fib[1]->devs[0]")
    assert pattern.search("skb_ctx *c") and not pattern.search("skb_flow_set_fibers(fl)")
    found = {name: sorted(set(m.group(0) for m in pattern.finditer(_source(name)))) for name in FLOW_MODULES}
    found = {name: hits for name, hits in found.items() if hits}
    assert not found, f"flow modules that reach the evaluator context: {found}"


def _outside_namespace_skb(src):
    """The text of src outside every `namespace skb { ... }` block."""
    out, i = [], 0
    for m in re.finditer(r"\bnamespace\s+skb\s*\{", src):
        if m.start() < i:
            continue
        out.append(src[i:m.start()])
        depth, j = 1, m.end()
        while depth and j < len(src):
            depth += {"{": 1, "}": -1}.get(src[j], 0)
            j += 1
        i = j
    out.append(src[i:])
    return "".join(out)


def test_internal_header_defines_types_in_namespace_skb():
    outside = _outside_namespace_skb(_source("skb_internal.hpp"))
    # a definition has a body; `struct skb_fiber_params;` only declares the public type it refers to
    defined = re.findall(r"\b(?:struct|class)\s+(\w+)[^;{()]*\{", outside)
    assert not defined, f"skb_internal.hpp defines {defined} outside namespace skb"
    assert _outside_namespace_skb("namespace skb { struct A { int x; }; } struct B {};").strip() == "struct B {};"
