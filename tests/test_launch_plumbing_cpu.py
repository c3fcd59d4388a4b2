"""Every kernel of libgm_b200.so is launched, counted, checked and profiled by one function, `launch` in engine.cu.

These checks read the C host sources: a call site that bypasses the launcher, counts launches by hand or leaves error
checking to a trailing cudaGetLastError would make gm_launch_count or the entry point's return code wrong again."""
import os
import re

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "generative-models_b200", "gm_b200", "csrc")


def _sources():
    return {f: open(os.path.join(CSRC, f)).read() for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".inl"))}


def _body(src, start):
    """The brace-delimited body of the definition that starts at `start`."""
    i = src.index("{", start)
    depth = 0
    for j in range(i, len(src)):
        depth += {"{": 1, "}": -1}.get(src[j], 0)
        if depth == 0:
            return src[i:j + 1]
    raise AssertionError("unbalanced braces")


def _launcher():
    src = _sources()["engine.cu"]
    m = re.search(r"\[\[nodiscard\]\] static int launch\(gm_ctx\* c,", src)
    assert m, "engine.cu defines `[[nodiscard]] static int launch(gm_ctx* c, ...)`"
    return _body(src, m.start())


def test_one_launch_call():
    hits = [(f, n) for f, s in _sources().items() for n in [s.count("cudaLaunchKernelEx")] if n]
    assert hits == [("engine.cu", 1)], hits
    assert "cudaLaunchKernelEx" in _launcher()


def test_launch_counter_changes_in_the_launcher_only():
    launcher = _launcher()
    assert "c->launches++" in launcher
    write = re.compile(r"(->|\.)launches\s*(\+\+|--|[-+*]?=(?!=))|(\+\+|--)\s*[\w>.-]*(->|\.)launches\b")
    for f, s in _sources().items():
        s = s.replace(launcher, "") if f == "engine.cu" else s
        for line in s.splitlines():
            if write.search(line):
                # the one other write: gm_launch_count's reset
                assert line.strip() == "if (reset) c->launches = 0;", (f, line)


def test_no_trailing_last_error_checks():
    for f, s in _sources().items():
        assert not re.search(r"CU_OK\([^;]*cudaGetLastError\(\)", s), f
    # the launcher clears a failed launch's error; nothing else reads the runtime's last error
    calls = [(f, s.count("cudaGetLastError()")) for f, s in _sources().items() if "cudaGetLastError()" in s]
    assert calls == [("engine.cu", 1)] and "cudaGetLastError()" in _launcher(), calls


def test_no_process_wide_attribute_guard():
    # a process-wide `static bool` in front of cudaFuncSetAttribute sets the attribute on the first device only
    for f, s in _sources().items():
        lines = s.splitlines()
        for i, line in enumerate(lines):
            if re.search(r"\bstatic\s+bool\s+\w+\s*(=[^;]*)?;", line):
                assert not any("cudaFuncSetAttribute" in l for l in lines[i:i + 6]), (f, i + 1, line)
