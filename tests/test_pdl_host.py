"""Programmatic dependent launch (PDL), checked on the source.

Kernels launched through launch_k (common.cuh) carry cudaLaunchAttributeProgrammaticStreamSerialization: the next
kernel's CTAs may start while this one still runs, and only griddepcontrol.wait (pdl_wait()) orders a kernel after its
predecessors.  So every such kernel must call pdl_wait() before it touches global memory through a pointer argument,
and before its first `return`: a grid whose CTAs all exit without waiting completes early and lets its own dependents
overtake its predecessors.  This test parses mickey_b200/csrc and checks both rules for every kernel launched through
launch_k.  Kernels launched with <<<>>> run in plain stream order and are listed separately.
"""
import os
import re

from tests.common import ROOT

CSRC = os.path.join(ROOT, "mickey_b200", "csrc")
# launched with <<<>>> (no PDL attribute): a plain launch starts only after its predecessor has completed
PLAIN_LAUNCHES = {"patch_gather_kernel", "attention_kernel", "ingest_u8_kernel", "pose_to_submission_kernel",
                  "sampler_phist_kernel", "seed_set_kernel", "seed_advance_kernel"}


def read_sources():
    return {f: open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))}


def strip_comments(src):
    return re.sub(r"//[^\n]*|/\*.*?\*/", " ", src, flags=re.S)


def _close(s, i):
    """s[i] is an opening bracket: index just past its partner."""
    pairs = {"(": ")", "{": "}", "[": "]"}
    depth, want = 0, pairs[s[i]]
    for j in range(i, len(s)):
        if s[j] == s[i]:
            depth += 1
        elif s[j] == want:
            depth -= 1
            if depth == 0:
                return j + 1
    raise ValueError("unbalanced")


def kernel_definitions(sources):
    """{name: (parameter list, body)} of every __global__ function with a body."""
    out = {}
    for src in sources.values():
        src = strip_comments(src)
        for m in re.finditer(r"\b__global__\b", src):
            i = m.end()
            while True:
                i += len(src[i:]) - len(src[i:].lstrip())
                if src.startswith("void", i):
                    i += 4
                elif src.startswith("__launch_bounds__", i):
                    i = _close(src, src.index("(", i))
                else:
                    break
            name = re.match(r"\w+", src[i:]).group(0)
            p = src.index("(", i)
            pe = _close(src, p)
            b = pe + len(src[pe:]) - len(src[pe:].lstrip())
            if src[b] != "{":
                continue                                    # declaration only
            out[name] = (src[p + 1:pe - 1], src[b + 1:_close(src, b) - 1])
    return out


def launched(sources):
    """(names launched through launch_k, names launched with <<<>>>), template arguments dropped."""
    pdl, plain = set(), set()
    for f, src in sources.items():
        src = strip_comments(src)
        if f == "common.cuh":
            continue
        pdl |= set(re.findall(r"\blaunch_k\(\s*(\w+)", src))
        plain |= set(re.findall(r"\b(\w+)\s*(?:<[^<>;()]*>)?\s*<<<", src))
    return pdl, plain


def pointer_params(params):
    names, depth, cur = [], 0, ""
    for ch in params + ",":
        if ch in "(<[":
            depth += 1
        elif ch in ")>]":
            depth -= 1
        if ch == "," and depth == 0:
            if "*" in cur:
                names.append(re.findall(r"\w+", cur)[-1])
            cur = ""
        else:
            cur += ch
    return names


def accesses(body, name):
    """Offsets in `body` where pointer `name` is dereferenced or handed to a call (a load, a store, a helper)."""
    n = re.escape(name)
    pats = [rf"\b{n}\s*\[", rf"\*\s*\(?\s*{n}\b", rf"\b{n}\s*->", rf"[(,]\s*{n}\s*[+,)]"]
    return sorted(m.start() for p in pats for m in re.finditer(p, body))


def violations(sources):
    """[(kernel, problem)] of every launch_k kernel that breaks a rule."""
    defs = kernel_definitions(sources)
    pdl, _ = launched(sources)
    bad = []
    for name in sorted(pdl):
        assert name in defs, f"launch_k({name}) has no __global__ definition in csrc/"
        params, body = defs[name]
        w = body.find("pdl_wait()")
        if w < 0:
            bad.append((name, "never calls pdl_wait()"))
            continue
        r = re.search(r"\breturn\b", body)
        if r and r.start() < w:
            bad.append((name, "returns before pdl_wait()"))
        for p in pointer_params(params):
            a = accesses(body, p)
            if a and a[0] < w:
                bad.append((name, f"touches pointer argument {p} before pdl_wait()"))
    return bad


def test_every_launch_k_kernel_waits_before_it_returns_or_touches_memory():
    sources = read_sources()
    pdl, plain = launched(sources)
    assert len(pdl) >= 20, sorted(pdl)
    assert violations(sources) == []


def test_plain_launches_are_the_listed_ones():
    _, plain = launched(read_sources())
    assert plain == PLAIN_LAUNCHES, sorted(plain ^ PLAIN_LAUNCHES)


def body_start(src, kernel):
    """Offset just inside the opening brace of `kernel`'s definition in the raw source."""
    g = src.index("__global__", src.index(kernel) - 400)
    p = src.index("(", src.index(kernel, g))
    return src.index("{", _close(src, p)) + 1


def test_a_deleted_pdl_wait_is_reported():
    sources = read_sources()
    for kernel, f in (("linattn_kv_kernel", "head_ops.cu"), ("ransac_solve_kernel", "ransac.cu"),
                      ("mutual_strips_kernel", "matches.cu")):
        src = sources[f]
        w = src.index("pdl_wait();", body_start(src, kernel))
        broken = dict(sources, **{f: src[:w] + src[w + len("pdl_wait();"):]})
        found = violations(broken)
        assert found and all(k == kernel for k, _ in found), (kernel, found)


def test_an_early_return_and_an_early_read_are_reported():
    sources = read_sources()
    f, kernel = "head_ops.cu", "linattn_kv_kernel"
    src = sources[f]
    ptr = pointer_params(kernel_definitions(sources)[kernel][0])[0]
    at = body_start(src, kernel)
    for inject, what in (("if (threadIdx.x > 4096) return;\n", "returns before"),
                         (f"float early_ = (float){ptr}[0]; (void)early_;\n", f"pointer argument {ptr}")):
        broken = dict(sources, **{f: src[:at] + inject + src[at:]})
        assert [msg for k, msg in violations(broken) if what in msg] and all(k == kernel for k, _ in violations(broken)), what
