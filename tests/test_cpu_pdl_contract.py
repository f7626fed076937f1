"""CPU: the programmatic-dependent-launch contract of the kernels, read from kandinsky-2_b200/csrc/*.cu.

With tuning key 4 on, launch_k (k2_internal.h) lets kernel N start while kernel N-1 of the stream drains.  That is only safe
because every such kernel executes griddepcontrol.wait (pdl_wait) before it lets its own successor start
(griddepcontrol.launch_dependents, pdl_launch): kernel N then starts only after N-1 has waited for N-2, so launches N-2 and
earlier are complete.  What kernel N reads before its wait must not be produced by N-1.  A launch joined in from another
stream by an event wait is a full dependency, eagerly and under stream capture (tests/test_gpu_pdl_plans.py checks it).
This file checks, for every kernel launched through launch_k:

  - it calls pdl_wait();
  - every pdl_launch() comes after the first pdl_wait();
  - the global loads before pdl_wait() -- an __ldg, or an indexed / dereferenced pointer parameter or pointer member of a
    parameter struct -- are in _EARLY_LOADS below, each with its reason.  An allow-list entry no kernel uses any more fails
    too, so the list stays the list of what the kernels actually do.

The last tests plant violations into an in-memory copy of the sources and check the audit reports them."""
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "kandinsky-2_b200", "csrc")

# (kernel, pointer) -> why it may be read before pdl_wait()
_EARLY_LOADS = {
    ("gn_apply_kernel", "gamma"): "GroupNorm gain: a layer weight, written when the model is packed, never by a plan launch",
    ("gn_apply_kernel", "beta"): "GroupNorm bias: a layer weight, written when the model is packed, never by a plan launch",
    ("gn_apply_kernel", "film"): "FiLM rows: written by the forked branch, whose event join is a full dependency even in "
                                 "front of a PDL launch (tests/test_gpu_pdl_plans.py)",
}


def _sources():
    out = {}
    for path in sorted(glob.glob(os.path.join(CSRC, "*.cu"))):
        with open(path) as f:
            out[os.path.basename(path)] = f.read()
    return out


def _strip_comments(s):
    s = re.sub(r"/\*.*?\*/", lambda m: re.sub(r"[^\n]", " ", m.group(0)), s, flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def _match(s, i, open_, close):
    """Index one past the bracket that closes the one at s[i]."""
    depth = 0
    for j in range(i, len(s)):
        if s[j] == open_:
            depth += 1
        elif s[j] == close:
            depth -= 1
            if depth == 0:
                return j + 1
    raise AssertionError(f"unbalanced {open_}{close} at offset {i}")


def _split_top(s):
    """s split at the commas outside (), <>, [] and {}."""
    parts, depth, cur = [], 0, []
    for ch in s:
        if ch in "(<[{":
            depth += 1
        elif ch in ")>]}":
            depth -= 1
        if ch == "," and depth == 0:
            parts.append("".join(cur))
            cur = []
        else:
            cur.append(ch)
    parts.append("".join(cur))
    return [p.strip() for p in parts]


def _kernels(srcs):
    """{kernel name: (file, parameter list, body)} of every __global__ function."""
    out = {}
    for fname, src in srcs.items():
        for m in re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\s*\([^)]*\)\s*)?(\w+)\s*\(", src):
            p0 = m.end() - 1
            p1 = _match(src, p0, "(", ")")
            b0 = src.index("{", p1)
            out[m.group(1)] = (fname, src[p0 + 1:p1 - 1], src[b0 + 1:_match(src, b0, "{", "}") - 1])
    return out


def _structs(srcs):
    """{struct name: pointer member names} of the parameter structs."""
    out = {}
    for src in srcs.values():
        for m in re.finditer(r"\bstruct\s+(\w+)\s*\{", src):
            body = src[m.end():_match(src, m.end() - 1, "{", "}") - 1]
            out[m.group(1)] = set(re.findall(r"\*\s*(?:__restrict__\s+)?(\w+)\s*(?:[;,\[])", body))
    return out


def _launched(srcs, kernels):
    """{kernel name: file} of every kernel passed to launch_k.  The first argument may be a kernel, a template instance
    (conv_gemm_kernel<BN, ES>), a ternary between instances, or the parameter of a lambda that the file calls with kernels
    (k2_norm.cu: go(gn_apply_kernel<0, true>))."""
    out = {}
    for fname, src in srcs.items():
        for m in re.finditer(r"\blaunch_k\s*\(", src):
            args = src[m.end():_match(src, m.end() - 1, "(", ")") - 1]
            first = _split_top(args)[0]
            names = [w for w in re.findall(r"[A-Za-z_]\w*", first) if w in kernels]
            if not names and re.fullmatch(r"\w+", first):
                for lam in re.finditer(r"(\w+)\s*=\s*\[[^\]]*\]\s*\(\s*auto\s+" + first + r"\s*\)", src):
                    for call in re.finditer(r"\b" + lam.group(1) + r"\s*\(\s*([A-Za-z_]\w*)", src):
                        if call.group(1) in kernels:
                            names.append(call.group(1))
            assert names, f"{fname}: cannot tell which kernel launch_k({first}, ...) launches"
            for n in names:
                out[n] = fname
    return out


def _early_loads(params, head, structs):
    """Pointers loaded from global memory in `head` (the code before pdl_wait): __ldg arguments, indexed or dereferenced
    pointer parameters, and indexed pointer members of by-value parameter structs."""
    found = set()
    for m in re.finditer(r"__ldg\s*\(", head):
        arg = head[m.end():]
        arg = re.sub(r"^\s*(?:reinterpret_cast|static_cast)\s*<[^>]*>\s*\(", "", arg)
        chain = re.match(r"\s*(\w+(?:\s*(?:\.|->)\s*\w+)*)", arg)
        found.add(re.split(r"\.|->", chain.group(1))[-1].strip() if chain else "?")
    for p in _split_top(params):
        name = re.search(r"(\w+)\s*$", p)
        if not name:
            continue
        name = name.group(1)
        if "*" in p:
            if re.search(r"\b" + name + r"\s*\[", head) or re.search(r"(?:^|[=(,;{?:])\s*\*\s*" + name + r"\b", head):
                found.add(name)
        else:
            stype = re.findall(r"\w+", p)[-2] if len(re.findall(r"\w+", p)) >= 2 else ""
            for member in structs.get(stype, ()):
                if re.search(r"\b" + name + r"\s*\.\s*" + member + r"\s*\[", head) or \
                        re.search(r"\*\s*" + name + r"\s*\.\s*" + member + r"\b", head):
                    found.add(member)
    return found


def _audit(srcs):
    srcs = {k: _strip_comments(v) for k, v in srcs.items()}
    kernels = _kernels(srcs)
    structs = _structs(srcs)
    launched = _launched(srcs, kernels)
    no_wait, launch_first, early = [], [], {}
    for name in sorted(launched):
        _, params, body = kernels[name]
        w = body.find("pdl_wait()")
        if w < 0:
            no_wait.append(name)
            continue
        if any(m.start() < w for m in re.finditer(r"pdl_launch\s*\(\s*\)", body)):
            launch_first.append(name)
        for ptr in _early_loads(params, body[:w], structs):
            early[(name, ptr)] = launched[name]
    return dict(launched=launched, no_wait=no_wait, launch_first=launch_first, early=early)


@pytest.fixture(scope="module")
def audit():
    return _audit(_sources())


def test_the_audit_sees_every_pdl_kernel_family(audit):
    """The parser finds the launches it must find: plain, templated, ternary and lambda-forwarded first arguments."""
    for k in ("conv_gemm_kernel", "splitk_finalize_kernel", "attention_d64_kernel", "flash_attention_kernel", "gn_stats_kernel",
              "gn_finalize_kernel", "gn_apply_kernel", "sn_apply_kernel", "transpose_f16_kernel", "linear_kernel",
              "timestep_embedding_kernel", "stem_im2col_kernel", "step_begin_kernel", "step_end_kernel", "sampler_x0_kernel",
              "sampler_percentile_kernel", "sampler_post_kernel", "plms_step_kernel", "dpm_solver_step_kernel",
              "unipc_step_kernel"):
        assert k in audit["launched"], k


def test_every_pdl_kernel_waits(audit):
    assert audit["no_wait"] == [], f"launched through launch_k without pdl_wait(): {audit['no_wait']}"


def test_pdl_launch_comes_after_pdl_wait(audit):
    assert audit["launch_first"] == [], f"pdl_launch() before pdl_wait(): {audit['launch_first']}"


def test_loads_before_pdl_wait_are_allow_listed(audit):
    found = set(audit["early"])
    assert not found - set(_EARLY_LOADS), f"global loads before pdl_wait() not in the allow-list: {sorted(found - set(_EARLY_LOADS))}"
    assert not set(_EARLY_LOADS) - found, f"allow-list entries no kernel needs any more: {sorted(set(_EARLY_LOADS) - found)}"


def _plant(srcs, fname, kernel, old, new):
    """srcs with the first `old` inside `kernel`'s definition in `fname` replaced by `new`."""
    src = srcs[fname]
    at = re.search(r"\b" + kernel + r"\s*\(", src).start()
    i = src.index(old, at)
    return dict(srcs, **{fname: src[:i] + new + src[i + len(old):]})


def test_audit_reports_a_launch_before_the_wait():
    srcs = _plant(_sources(), "k2_misc.cu", "sampler_post_kernel", "pdl_wait();\n  pdl_launch();", "pdl_launch();\n  pdl_wait();")
    assert _audit(srcs)["launch_first"] == ["sampler_post_kernel"]


def test_audit_reports_a_missing_wait():
    srcs = _plant(_sources(), "k2_movq.cu", "transpose_f16_kernel", "pdl_wait();", "")
    assert _audit(srcs)["no_wait"] == ["transpose_f16_kernel"]


@pytest.mark.parametrize("fname,kernel,line,ptr", [
    ("k2_norm.cu", "gn_apply_kernel", "const __half early = __ldg(p.s0);", "s0"),                  # activation, struct member
    ("k2_misc.cu", "linear_kernel", "const float early = x[lane];", "x"),                         # pointer parameter
    ("k2_misc.cu", "step_end_kernel", "const int early = *counter;", "counter"),                  # dereference
    ("k2_movq.cu", "sn_apply_kernel", "const float early = p.zq[n];", "zq"),                      # indexed struct member
])
def test_audit_reports_an_activation_read_before_the_wait(fname, kernel, line, ptr):
    srcs = _plant(_sources(), fname, kernel, "pdl_wait();", line + "\n  pdl_wait();")
    early = _audit(srcs)["early"]
    assert (kernel, ptr) in early and (kernel, ptr) not in _EARLY_LOADS
