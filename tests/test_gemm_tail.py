"""The wgmma GEMM with its split drain of the CTA's last tile (gemm_sm90.cuh) compiles for sm_90a, with the build's own
flags, to 0 spill bytes and no stack frame in every instantiation the launcher dispatches, within the 384 x 168
registers of the launch (40 for the producer warpgroup, 232 for each consumer warpgroup after setmaxnreg), and without
wgmma serialisation (ptxas warnings C7510 / C7512).  Runs on the CPU."""
import re
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent


def test_gemm_instantiations_compile_without_spills(tmp_path):
    from f5_tts_mlx_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-cubin", str(ROOT / "f5_tts_mlx_b200" / "csrc" / "gemm.cu"), "-o",
           str(tmp_path / "gemm.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    log = r.stdout + r.stderr
    assert not re.search(r"C751[02]|serialized", log), re.findall(r".*serialized.*", log)[:4]
    found = {}
    for m in re.finditer(r"Compiling entry function '(\S+)'(.*?)Used (\d+) registers", log, re.S):
        if "gemm_bf16_tn_kernel" in m[1]:
            spill = sum(int(x) for x in re.findall(r"(\d+) bytes spill (?:stores|loads)", m[2]))
            stack = sum(int(x) for x in re.findall(r"(\d+) bytes stack frame", m[2]))
            found[m[1]] = (spill, stack, int(m[3]))
    assert len(found) == 36, sorted(found)        # 2 widths x (14 of dispatch_epi + 4 of dispatch_scaled)
    bad = {k: v for k, v in found.items() if v[0] or v[1] or v[2] > 168}
    assert not bad, bad
