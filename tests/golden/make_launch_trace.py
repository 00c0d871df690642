"""Launch trace of the DiT, UNetT, ODE sampler and duration predictor host code, made on the CPU;
launch_trace_digests.txt.

csrc/dit.cu, csrc/unett.cu and csrc/duration.cu hold no kernels.  Compiled with the library's nvcc flags and linked against
tests/host_trace/stubs.cu instead of the rest of the library, they run without a GPU, and every launch they make is
printed with all of its arguments (see stubs.cu for the cases).  The full trace is about 2 MB of text, so the fixture
keeps one line per case: the first 16 hex digits of the SHA-256 of the case's trace (its header, every launch line
and every return code), its number of calls and its header.  tests/test_host_launch_trace.py rebuilds the trace from
the working tree and requires every digest to match, so a change to this host code that alters what it launches, in
any mode, shows up on the CPU.

    python tests/golden/make_launch_trace.py                 # rewrites the fixture (only for a change meant to
                                                             # launch different work)
    python tests/golden/make_launch_trace.py --show 'TEXT'   # prints the full trace of the cases whose header
                                                             # contains TEXT (run it at two commits and diff)
"""
import hashlib
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

FIXTURE = os.path.join(HERE, "launch_trace_digests.txt")
SOURCES = [os.path.join(ROOT, "f5_tts_mlx_b200", "csrc", "dit.cu"),
           os.path.join(ROOT, "f5_tts_mlx_b200", "csrc", "duration.cu"),
           os.path.join(ROOT, "f5_tts_mlx_b200", "csrc", "unett.cu"),
           os.path.join(ROOT, "tests", "host_trace", "stubs.cu")]


def launch_trace() -> str:
    """Compiles the host code against the recording stubs in a temporary directory and returns its trace."""
    from f5_tts_mlx_b200 import build
    flags = [f for f in build.NVCC_FLAGS if f not in ("-Xptxas=-v", "-lineinfo")]
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "launch_trace")
        r = subprocess.run([build._nvcc(), *flags, *SOURCES, "-o", exe], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed on the launch-trace program:\n" + r.stdout + r.stderr)
        r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
        if r.returncode != 0:
            raise RuntimeError(f"the launch-trace program exited with {r.returncode}:\n{r.stderr}")
        return r.stdout


def cases(trace: str) -> list[tuple[str, list[str]]]:
    """(header, lines) of every case; a case starts at a line beginning with '== '"""
    out = []
    for line in trace.splitlines():
        if line.startswith("== "):
            out.append((line[3:], []))
        else:
            out[-1][1].append(line)
    return out


def digest_line(header: str, lines: list[str]) -> str:
    h = hashlib.sha256("\n".join([header, *lines]).encode()).hexdigest()[:16]
    calls = sum(1 for l in lines if l.startswith("  "))
    return f"{h} {calls:3d} {header}"


if __name__ == "__main__":
    trace = launch_trace()
    if len(sys.argv) == 3 and sys.argv[1] == "--show":
        for header, lines in cases(trace):
            if sys.argv[2] in header:
                print("== " + header, *lines, sep="\n")
        sys.exit(0)
    digests = [digest_line(h, l) for h, l in cases(trace)]
    with open(FIXTURE, "w") as f:
        f.write("\n".join(digests) + "\n")
    print(f"wrote {FIXTURE}: {len(digests)} cases of {trace.count(chr(10))} trace lines")
