"""The machine code of the forward tile kernel keeps the schedule DESIGN.md §3.2 describes: in the steady-state loop,
tile j's exponentials are issued after the wait for S_j (`WARPGROUP.DEPBAR.LE gsb0, 0x1`) and before the wait for
O += P_{j-1} V_{j-1} (`WARPGROUP.DEPBAR.LE gsb0, 0x0`), so they run while that GEMM is on the tensor cores, and each
is issued once (64 per thread and tile, plus the two of the row rescale). Left to itself, ptxas hoists the PV wait
above the exponentials, and it if-converted the masked and unmasked forms into two predicated copies of every one.
A compiler upgrade could bring either back without changing a result, so this reads the SASS of the built library."""
import bisect
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "lwm_b200", "lib", "liblwm_b200.so")

# attn_fwd_kernel<kF16, kInfer, kMap>
INSTANCES = {
    "bf16": "_ZN3lwm15attn_fwd_kernelILb0ELb0ELb0EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
    "fp16": "_ZN3lwm15attn_fwd_kernelILb1ELb0ELb0EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
    "bf16_map": "_ZN3lwm15attn_fwd_kernelILb0ELb0ELb1EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
    "fp16_map": "_ZN3lwm15attn_fwd_kernelILb1ELb0ELb1EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
    "infer": "_ZN3lwm15attn_fwd_kernelILb1ELb1ELb0EEEv14CUtensorMap_stS1_S1_NS_9FwdParamsE",
}

_INSN = re.compile(r"/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
_COND_BRA = re.compile(r"^@!?U?P\w+\s+BRA(?:\.\S+)?\s+0x([0-9a-f]+)")
_HGMMA_SS = re.compile(r"HGMMA\.\S+\s+R\d+,\s+gdesc")         # S = Q K^T: both operands in shared memory
_HGMMA_RS = re.compile(r"HGMMA\.\S+\s+R\d+,\s+R\d+,\s+gdesc")  # O += P V: P from registers


def _cuobjdump():
    tool = shutil.which("cuobjdump")
    if tool is None:
        tool = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    return tool if os.path.exists(tool) else None


@pytest.fixture(scope="module")
def sass():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs cuobjdump and the built liblwm_b200.so")
    r = subprocess.run([tool, "-sass", "-fun", ",".join(INSTANCES.values()), LIB], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    fns, cur = {}, None
    for line in r.stdout.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = fns.setdefault(m.group(1), [])
            continue
        m = _INSN.search(line)
        if m and cur is not None:
            cur.append((int(m.group(1), 16), m.group(2)))
    return fns


def _steady_state_loop(insns):
    """the instructions of the innermost loop that issues both the S and the PV GEMMs: the shortest address range
    [target, branch] of a conditional backward branch that holds both kinds of HGMMA"""
    addrs = [a for a, _ in insns]
    ss = [a for a, t in insns if _HGMMA_SS.search(t)]
    rs = [a for a, t in insns if _HGMMA_RS.search(t)]
    best = None
    for i, (addr, text) in enumerate(insns):
        m = _COND_BRA.match(text)
        if not m or int(m.group(1), 16) >= addr:
            continue
        lo = int(m.group(1), 16)
        if any(lo <= a <= addr for a in ss) and any(lo <= a <= addr for a in rs):
            if best is None or addr - lo < best[1] - best[0]:
                best = (lo, addr)
    if best is None:
        return None
    return insns[bisect.bisect_left(addrs, best[0]):bisect.bisect_right(addrs, best[1])]


@pytest.mark.parametrize("instance", sorted(INSTANCES))
def test_exponentials_run_under_the_pv_gemm(sass, instance):
    insns = sass.get(INSTANCES[instance])
    assert insns, "attn_fwd_kernel instance %s not in the library" % instance
    loop = _steady_state_loop(insns)
    assert loop is not None, "no loop issues both the S and the PV wgmma"
    texts = [t for _, t in loop]
    s_ready = next(i for i, t in enumerate(texts) if "WARPGROUP.DEPBAR.LE gsb0, 0x1" in t)
    pv_done = next(i for i in range(s_ready, len(texts)) if "WARPGROUP.DEPBAR.LE gsb0, 0x0" in texts[i])
    under_pv = sum("MUFU.EX2" in t for t in texts[s_ready:pv_done])
    in_loop = sum("MUFU.EX2" in t for t in texts)
    assert under_pv >= 64, "%d exponentials between the S wait and the PV wait" % under_pv
    assert in_loop <= 66, "%d exponentials in the loop: some are issued twice" % in_loop
