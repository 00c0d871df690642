"""The DiT, ODE sampler and duration predictor host code launches exactly the work the committed digests record: the
same launches in the same order with the same arguments, every f5_gemm_args field included, in each of the five DiT
modes, with and without CFG, each drop_flags value, seq_len and valid_len bound or not, on both sides of the weight
prefetch cutoff, for the three solvers, and the same refusals of partly bound modes.  Runs on the CPU: the host code
is linked against recording stubs (tests/host_trace/stubs.cu, tests/golden/make_launch_trace.py)."""
import importlib.util
import os


def _make_launch_trace(golden_dir):
    spec = importlib.util.spec_from_file_location("make_launch_trace", os.path.join(golden_dir, "make_launch_trace.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_launch_trace_matches_fixture(golden_dir):
    mod = _make_launch_trace(golden_dir)
    got = mod.cases(mod.launch_trace())
    with open(mod.FIXTURE) as f:
        want = f.read().splitlines()
    assert [h for h, _ in got] == [w.split(None, 2)[2] for w in want], "the set or order of cases changed"
    for (header, lines), w in zip(got, want):
        if mod.digest_line(header, lines) != w:
            raise AssertionError(
                f"case `{header}` launches different work than the fixture records ({w.split()[1]} calls there).  "
                f"What it launches now is below; `python tests/golden/make_launch_trace.py --show '{header}'` at the "
                "parent commit prints what it launched there.\n" + "\n".join(lines))
