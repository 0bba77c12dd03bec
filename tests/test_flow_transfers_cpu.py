"""Static CPU test of the host-array calls under skellysim_b200/csrc: the flow and skb_mflow describe their copies with
one set of transfer types (skb_flow.hpp) and move them by one path, and the flow keeps no per-purpose staging buffers
beside its device workspace.  Reads the sources only: needs no library and no GPU."""
import glob
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "skellysim_b200", "csrc")

# the per-purpose staging buffers the flow's host-array calls once used (some of them also as device workspace)
REMOVED_FIELDS = ["in_fib", "in_shell", "in_body", "in_force", "in_torque", "x_fib", "res_fib", "res_shell", "vb",
                  "sys_x", "sys_y"]


def _source(path):
    """The file without comments and string literals."""
    src = open(path if os.path.isabs(path) else os.path.join(CSRC, path)).read()
    return re.sub(r'//[^\n]*|/\*.*?\*/|"(?:\\.|[^"\\\n])*"', " ", src, flags=re.S)


def _struct_body(src, name):
    """The text between the braces of `struct name { ... }`."""
    m = re.search(r"\bstruct\s+" + name + r"\s*\{", src)
    assert m, f"struct {name} not found"
    depth, j = 1, m.end()
    while depth:
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        j += 1
    return src[m.end():j - 1]


def test_the_flow_declares_no_staging_buffers():
    body = _struct_body(_source("skb_flow.hpp"), "skb_flow")
    assert re.search(r"\bDevBuf\s+vel\b", body), "the reader no longer finds the flow's workspace"
    found = [f for f in REMOVED_FIELDS if re.search(r"\b%s\b" % f, body)]
    assert not found, f"skb_flow declares staging buffers {found}"


def test_transfer_types_are_defined_once_in_the_flow_header():
    defs = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "*.*"))):
        for m in re.finditer(r"\bstruct\s+(Run|Transfer|Transfers)\s*\{", _source(path)):
            defs.setdefault(m.group(1), []).append(os.path.basename(path))
    assert defs == {"Run": ["skb_flow.hpp"], "Transfer": ["skb_flow.hpp"], "Transfers": ["skb_flow.hpp"]}, defs


def test_host_forms_write_no_copies_of_their_own():
    # the flow's free upload / download helpers; a member such as ops.upload(...) is another thing
    call = re.compile(r"(?<![\w.>])(?:upload|download)\s*\(")
    assert call.search("SKB_TRY(upload(fl, buf, h, n));") and call.search("return download(fl, h, b, n);")
    assert not call.search("fl->ops.upload(own, A)") and not call.search("rhs_items.upload(p, n, st)")
    for name in ("skb_matvec.cu", "skb_system.cu"):
        hits = call.findall(_source(name))
        assert not hits, f"{name} calls {hits}"


def test_mflow_has_no_copy_loop_of_its_own():
    src = _source("skb_mflow.cu")
    copies = re.findall(r"cudaMemcpyHostToDevice|cudaMemcpyDeviceToHost|cudaMemcpyDefault", src)
    assert not copies, f"skb_mflow.cu copies between host and device itself: {copies}"
    assert re.search(r"\bstage_slots\s*\(", src) and re.search(r"\bissue\s*\(", src)
