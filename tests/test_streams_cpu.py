"""Static check that every device write of the library is ordered on a stream it chooses: no CUDA call in csrc/ enqueues on
the legacy default stream or waits for the whole device, outside a short allowlist of debug functions.

Why: torch.cuda.Stream() streams are non-blocking, so nothing orders them against the legacy default stream.  A memset or copy
that the library issues there, while a caller runs on its own stream (a collector beside a learner busy on the default stream),
lands whenever the default stream gets to it: after the kernels on the caller's stream that read what it writes.  The per-step
entry points enqueue on the stream they are given; the setup entry points write on the library's setup stream and wait for it
(setup_memset / setup_upload, lz_common.cuh).  tests/test_gpu_streams.py runs both on an H100 next to a busy default stream.

Flagged, with the function that contains it:
  - the stream-less copies and memsets (cudaMemset(, cudaMemcpy(, cudaMemcpyToSymbol(, ...): they run on the legacy stream;
  - cudaDeviceSynchronize, and a synchronize of stream 0;
  - an async call (cudaMemsetAsync, cudaMemcpyAsync, cudaEventRecord, cudaGraphLaunch) without a stream argument or with the
    legacy stream as its stream;
  - a kernel launch <<<...>>> without a stream argument or with the legacy stream.
Needs no GPU and no compiler."""
import os
import re

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "lightzero_b200", "csrc")

# The calls that may stay, each pinned to its function and to the exact number of such calls there (one more of the same kind
# in the same function fails): debug paths, which read device state back on purpose
ALLOWED = {
    ("lz_debug_tc_stamps", "cudaMemcpy("): (1, "debug: copies the clock stamps of an instrumented launch to the host"),
    ("lz_tree_debug_rng", "cudaDeviceSynchronize"): (1, "debug: waits for the resets that bump the RNG epoch on the device"),
    ("lz_tree_debug_rng", "cudaMemcpy("): (1, "debug: reads the RNG epoch back"),
    ("tc_prepare_launch", "cudaMemset("): (1, "debug: zeroes the stamp buffer, allocated only with LZ_TC_DEBUG set"),
}

SYNC_CALLS = ("cudaMemset", "cudaMemset2D", "cudaMemset3D", "cudaMemcpy", "cudaMemcpy2D", "cudaMemcpy3D", "cudaMemcpyPeer",
              "cudaMemcpyToSymbol", "cudaMemcpyFromSymbol")
# async calls: number of arguments, the last one being the stream (the C++ API defaults it to 0 when left out)
ASYNC_CALLS = {"cudaMemsetAsync": 4, "cudaMemcpyAsync": 5, "cudaMemcpyToSymbolAsync": 6, "cudaMemcpyFromSymbolAsync": 6,
               "cudaEventRecord": 2, "cudaGraphLaunch": 2}
LEGACY = {"0", "nullptr", "NULL", "cudaStreamLegacy", "(cudaStream_t)0", "(cudaStream_t)nullptr"}


def strip(src):
    """Comments blanked and string / char literals emptied, newlines kept (so offsets still map to the same lines)."""
    out, i, n = [], 0, len(src)
    while i < n:
        c = src[i]
        if src.startswith("//", i):
            j = src.find("\n", i)
            j = n if j < 0 else j
            out.append(" " * (j - i)); i = j
        elif src.startswith("/*", i):
            j = src.find("*/", i + 2)
            j = n if j < 0 else j + 2
            out.append(re.sub(r"[^\n]", " ", src[i:j])); i = j
        elif c in "\"'":
            j = i + 1
            while j < n and src[j] != c:
                j += 2 if src[j] == "\\" else 1
            out.append(c + " " * (j - i - 1) + c); i = j + 1
        else:
            out.append(c); i += 1
    return "".join(out)


def _split_args(s):
    """Top-level comma split of an argument list (parentheses, brackets and braces nest)."""
    args, depth, cur = [], 0, []
    for c in s:
        if c in "([{":
            depth += 1
        elif c in ")]}":
            depth -= 1
        if c == "," and depth == 0:
            args.append("".join(cur).strip()); cur = []
        else:
            cur.append(c)
    if "".join(cur).strip():
        args.append("".join(cur).strip())
    return args


def _close(s, i, open_="(", close=")"):
    """Index of the bracket closing the one at s[i]."""
    depth = 0
    for j in range(i, len(s)):
        if s[j] == open_:
            depth += 1
        elif s[j] == close:
            depth -= 1
            if depth == 0:
                return j
    return len(s)


def _function_name(head):
    """The function a body belongs to, from the text between the previous ; { } and its opening brace (None: not a function)."""
    h = head.strip()
    if h.startswith("template"):                         # template <int C, int NT = 1>: its '=' is not an initializer's
        depth, i = 0, h.index("<")
        for i in range(i, len(h)):
            depth += {"<": 1, ">": -1}.get(h[i], 0)
            if depth == 0:
                break
        h = h[i + 1:].strip()
    if not h or re.match(r"(namespace|extern|struct|class|union|enum)\b", h) or "=" in h.split("(")[0] or "(" not in h:
        return None
    # the parameter list is the last top-level parenthesised group (earlier ones: __launch_bounds__(...), attributes)
    last, i = None, 0
    while i < len(h):
        if h[i] == "(":
            j = _close(h, i)
            last = i; i = j + 1
        else:
            i += 1
    m = re.search(r"([A-Za-z_]\w*)\s*$", h[:last])
    if not m or m.group(1) in ("if", "for", "while", "switch", "catch", "__launch_bounds__"):
        return None
    return m.group(1)


def functions(text):
    """Per character offset of a stripped source, the name of the enclosing function ('' at file scope)."""
    owner = [""] * len(text)
    stack, head_start, cur = [], 0, ""
    for i, c in enumerate(text):
        if c == "{":
            name = _function_name(text[head_start:i]) if not cur else None
            stack.append(name)
            if name:
                cur = name
            head_start = i + 1
        elif c == "}":
            if stack and stack.pop():
                cur = ""
            head_start = i + 1
        elif c == ";":
            head_start = i + 1
        owner[i] = cur
    return owner


def scan_source(src):
    """[(line, function, construct, text)] of the calls that this file's rules reject."""
    text = strip(src)
    owner = functions(text)
    line_of = lambda i: text.count("\n", 0, i) + 1
    found = []

    def hit(i, construct, what):
        found.append((line_of(i), owner[i], construct, what))

    for m in re.finditer(r"\b(%s)\s*\(" % "|".join(SYNC_CALLS), text):
        hit(m.start(), m.group(1) + "(", "stream-less %s (legacy default stream)" % m.group(1))
    for m in re.finditer(r"\bcudaDeviceSynchronize\b", text):
        hit(m.start(), "cudaDeviceSynchronize", "cudaDeviceSynchronize")
    for m in re.finditer(r"\bcudaStreamSynchronize\s*\(", text):
        args = _split_args(text[m.end():_close(text, m.end() - 1)])
        if not args or args[0].replace(" ", "") in LEGACY:
            hit(m.start(), "cudaStreamSynchronize(0)", "synchronize of the legacy default stream")
    for m in re.finditer(r"\b(%s)\s*\(" % "|".join(ASYNC_CALLS), text):
        args = _split_args(text[m.end():_close(text, m.end() - 1)])
        want = ASYNC_CALLS[m.group(1)]
        if len(args) < want or args[want - 1].replace(" ", "") in LEGACY:
            hit(m.start(), m.group(1), "%s on the legacy default stream" % m.group(1))
    for m in re.finditer(r"<<<", text):
        end = text.find(">>>", m.end())
        args = _split_args(text[m.end():end])
        kernel = re.search(r"([\w:]+(?:\s*<[^<>;]*>)?)\s*$", text[max(0, m.start() - 200):m.start()])
        if len(args) < 4 or args[3].replace(" ", "") in LEGACY:
            hit(m.start(), "<<<", "launch of %s without a stream" % (kernel.group(1) if kernel else "a kernel"))
    return sorted(found)


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh")))


def scan_tree(csrc=CSRC):
    """{(file, line, function, construct): text} over every .cu / .cuh in csrc."""
    out = {}
    for f in sorted(os.listdir(csrc)):
        if f.endswith((".cu", ".cuh")):
            with open(os.path.join(csrc, f)) as fh:
                for line, fn, construct, what in scan_source(fh.read()):
                    out[(f, line, fn, construct)] = what
    return out


def _hits():
    """{(function, construct): ["file:line: text", ...]} of every flagged call"""
    hits = {}
    for (f, line, fn, construct), what in scan_tree().items():
        hits.setdefault((fn, construct), []).append("%s:%d in %s(): %s" % (f, line, fn or "<file scope>", what))
    return hits


def _violations(hits):
    """the flagged calls past their function's allowance (every one, when a function has more than it is allowed)"""
    bad = []
    for key, sites in sorted(hits.items()):
        allowed = ALLOWED.get(key, (0, ""))[0]
        if len(sites) > allowed:
            bad += sites if not allowed else ["%d such calls, %d allowed: %s" % (len(sites), allowed, s) for s in sites]
    return bad


def test_no_legacy_stream_writes_outside_the_allowlist():
    bad = _violations(_hits())
    assert not bad, "device work outside the caller's stream or the setup stream:\n  " + "\n  ".join(bad)


def test_allowlist_is_pinned_to_the_number_of_calls():
    """a second stream-less memset in tc_prepare_launch (outside its LZ_TC_DEBUG branch, say) is not covered by the entry"""
    hits = {("tc_prepare_launch", "cudaMemset("): ["net_tc.cu:970", "net_tc.cu:975"], ("lz_tree_debug_rng", "cudaMemcpy("): ["t"]}
    assert len(_violations(hits)) == 2
    assert _violations({("tc_prepare_launch", "cudaMemset("): ["net_tc.cu:970"]}) == []


def test_allowlist_entries_are_still_needed():
    hits = _hits()
    stale = sorted("%s: %d allowed, %d found" % (key, n, len(hits.get(key, ())))
                   for key, (n, _) in ALLOWED.items() if len(hits.get(key, ())) != n)
    assert not stale, "allowlist counts that no longer match the sources (update or remove them): %s" % stale


def test_every_launch_site_was_seen():
    """The scanner parses every file: each launch it finds sits in a named function, and there are as many as the sources have."""
    launches = 0
    for f in _sources():
        with open(os.path.join(CSRC, f)) as fh:
            text = strip(fh.read())
        owner = functions(text)
        for m in re.finditer(r"<<<", text):
            assert owner[m.start()], "%s:%d: launch outside any function the scanner recognised" % (f, text.count("\n", 0, m.start()) + 1)
            launches += 1
    assert launches >= 40, launches


# ---- the scanner itself: each rule fires on its construct and only there ----
_WRAP = """namespace lz {
__global__ void __launch_bounds__(64)
k_a(int *p) { p[0] = 1; }
}  // namespace lz
extern "C" {
int entry(int *d, const int *h, lz_stream s_)
{
    cudaStream_t s = (cudaStream_t)s_;
    auto take = [&](size_t n) { return n; };
    if (d) {
        %s
    }
    return 0;
}
}
"""


@pytest.mark.parametrize("body, construct", [
    ("cudaMemset(d, 0, 4);", "cudaMemset("),
    ("LZ_CUDA_CHECK(cudaMemcpy(d, h, 4, cudaMemcpyHostToDevice));", "cudaMemcpy("),
    ("cudaMemcpyToSymbol(sym, h, 4);", "cudaMemcpyToSymbol("),
    ("cudaDeviceSynchronize();", "cudaDeviceSynchronize"),
    ("cudaStreamSynchronize(0);", "cudaStreamSynchronize(0)"),
    ("cudaStreamSynchronize(nullptr);", "cudaStreamSynchronize(0)"),
    ("cudaMemsetAsync(d, 0, 4);", "cudaMemsetAsync"),
    ("cudaMemcpyAsync(d, h, 4, cudaMemcpyHostToDevice, 0);", "cudaMemcpyAsync"),
    ("cudaEventRecord(ev);", "cudaEventRecord"),
    ("cudaGraphLaunch(exec, cudaStreamLegacy);", "cudaGraphLaunch"),
    ("k_a<<<1, 64>>>(d);", "<<<"),
    ("k_a<<<dim3(std::min(1, 2), 1), 64, 0>>>(d);", "<<<"),
    ("k_a<<<1, 64, 0, 0>>>(d);", "<<<"),
])
def test_scanner_flags(body, construct):
    found = scan_source(_WRAP % body)
    assert [(fn, c) for _, fn, c, _ in found] == [("entry", construct)], found
    assert found[0][0] == 11          # the line of the call


@pytest.mark.parametrize("body", [
    "k_a<<<dim3(std::min(1, 2), 1), 64, 0, s>>>(d);",
    "cudaMemsetAsync(d, 0, 4, s);",
    "cudaMemcpyAsync(d, h, 4, cudaMemcpyHostToDevice, (cudaStream_t)s_);",
    "cudaStreamSynchronize(s); cudaEventRecord(ev, s); cudaGraphLaunch(exec, s);",
    "// cudaMemset(d, 0, 4); cudaDeviceSynchronize();",
    "/* k_a<<<1, 64>>>(d); */ set_error(\"cudaMemcpy(d, h) failed\");",
])
def test_scanner_passes(body):
    assert scan_source(_WRAP % body) == []
