"""Static checks on the built library and the kernel sources (CPU only; cuobjdump cross-reads the sm_90a SASS):

  * the GEMM-shaped kernels are wgmma kernels (HGMMA in their SASS, operands staged by TMA) and contain no legacy HMMA;
  * the legacy tensor path (HMMA, mma.sync) appears ONLY in the three register-fragment kernels that use it on purpose
    (DESIGN.md 3: dla_front, stem_s2_mma, b3d_sparse);
  * the programmatic-dependent-launch rule of csrc/pdl.cuh: every kernel launched through launch_pdl() starts with
    DD3D_PDL_PROLOGUE() (otherwise it could touch memory an earlier kernel is still writing), and launch_pdl() itself sets the
    attribute only inside a PdlScope;
  * the double-buffer rule of the cp.async kernels: a prefetch is issued only after the barrier that retires the readers of
    the buffer it overwrites (stem_mma had it the other way round once; the race showed only at full size)."""
import glob
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
CSRC = os.path.join(ROOT, "dd3d_b200", "csrc")
SO = os.path.join(ROOT, "dd3d_b200", "_lib", "libdd3d_b200.so")


def _sass_by_kernel():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(SO):
        pytest.skip("cuobjdump or the built library is not available")
    out = subprocess.run([exe, "-sass", SO], capture_output=True, text=True, timeout=600).stdout
    kernels, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+(?:\.[A-Z0-9_.]+)?)", line)
        if m and cur:
            kernels[cur].append(m.group(1))
    return kernels


def test_tensor_core_paths_in_the_sass():
    kernels = _sass_by_kernel()
    assert len(kernels) > 30
    def has(ops, prefix):
        return any(o.startswith(prefix) for o in ops)
    tc = {n: o for n, o in kernels.items() if re.search(r"conv_igemm_kernel|conv_taps_kernel|stem_tc_kernel", n)}
    assert len(tc) >= 8  # 4 conv_igemm variants (generic / halo x bf16 / fp16) + 2 taps + 2 stems
    for n, ops in tc.items():
        assert has(ops, "HGMMA"), f"{n}: no wgmma"
        assert not has(ops, "HMMA"), f"{n}: legacy mma.sync in a wgmma kernel"
    for n, ops in kernels.items():
        if re.search(r"conv_igemm_kernel|conv_taps_kernel", n):
            assert has(ops, "UTMALDG"), f"{n}: operands are not staged by TMA"
        if re.search(r"conv_igemm_kernel", n):
            assert has(ops, "UTMASTG"), f"{n}: outputs are not stored by TMA"
    legacy = {n for n, ops in kernels.items() if has(ops, "HMMA")}
    assert legacy, "the register-fragment kernels are missing"
    for n in legacy:
        assert re.search(r"dla_front_kernel|stem_s2_mma_kernel|b3d_sparse_kernel", n), f"unexpected mma.sync kernel: {n}"
    stem = [o for n, o in kernels.items() if "stem_s2_mma_kernel" in n]
    assert stem and all(has(o, "STG.E.128") for o in stem), "stem_mma: 128-bit stores expected"



def test_wgmma_pipelines_are_not_serialized():
    """ptxas reports C7510 / C7520 when it serializes a kernel's wgmma pipeline (a call, or control flow it cannot prove
    warpgroup-uniform, between issue and wait): the build's ptxas logs must carry neither."""
    logs = sorted(glob.glob(os.path.join(ROOT, "dd3d_b200", "_lib", "obj", "*.ptxas.log")))
    if not logs:
        pytest.skip("the build's ptxas logs are not available")
    bad = []
    for path in logs:
        with open(path) as f:
            bad += [f"{os.path.basename(path)}: {line.strip()[:160]}" for line in f if re.search(r"\(C75(10|20)\)", line)]
    assert not bad, "\n".join(bad)

def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_pdl_rule_in_the_sources():
    pdl = _src("pdl.cuh")
    assert "g_pdl_scope_depth > 0" in pdl and "struct PdlScope" in pdl
    launched, defined = set(), {}
    for fn in sorted(os.listdir(CSRC)):
        if not fn.endswith(".cu"):
            continue
        s = _src(fn)
        for m in re.finditer(r"launch_pdl\(\s*([A-Za-z_0-9]+)", s):
            launched.add(m.group(1))
        for m in re.finditer(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?([A-Za-z_0-9]+)\s*\(", s):
            body = s[s.index("{\n", m.end()) + 2:]
            defined[m.group(1)] = body.lstrip().split("\n", 1)[0].strip()
    assert len(launched) >= 15, launched
    for k in launched:
        assert k in defined, f"{k}: definition not found"
        assert defined[k].startswith("DD3D_PDL_PROLOGUE();"), f"{k} is launched programmatically but does not start with the prologue"
    eng = _src("engine.cu")
    i_pre, i_scope, i_ops = eng.index('"preprocess");'), eng.index("PdlScope pdl_scope;"), eng.index("for (const Op& op : P.ops) {", eng.index("PdlScope pdl_scope;"))
    assert i_pre < i_scope < i_ops, "the scope must open after the first kernel of the forward and before the op loop"
    assert eng.count("PdlScope") == 1 and "PdlScope" not in _src("capi.cu"), "operator-level entry points never open a PdlScope"


@pytest.mark.parametrize("fn", ["stem_mma.cu", "dla_front.cu", "b3d_sparse.cu"])
def test_cp_async_prefetch_follows_the_barrier(fn):
    """In the tile / chunk loop of each cp.async kernel the first __syncthreads() precedes... or, where the prefetch comes first
    (dla_front, b3d_sparse), at least one more barrier separates the last reader of the buffer from the next iteration."""
    s = _src(fn)
    body = s[s.index("for (", s.index("cp.async.commit_group")):]
    i_sync, i_load = body.index("__syncthreads()"), min(i for i in (body.find("load_input("), body.find("stage_weights(")) if i >= 0)
    if i_load < i_sync:  # prefetch issued before the iteration's first barrier: legal only with later barriers in the same iteration
        assert body.count("__syncthreads()") >= 2, fn
    else:
        assert "wait_group" in body[:i_sync], fn
