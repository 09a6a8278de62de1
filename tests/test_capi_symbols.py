"""CPU suite: the C-ABI library builds for sm_90a, loads, exports every symbol include/tce_b200.h declares, and
refuses to compute without a GPU (no CPU fallback)."""
import ctypes as C
import re
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def built_lib():
    from tinychatengine_b200.build import build

    return build()


def declared_symbols():
    text = (ROOT / "include" / "tce_b200.h").read_text()
    return sorted(set(re.findall(r"TCE_API\s+[\w\s\*]+?\b(tce_\w+)\s*\(", text)))


def test_header_declares_something():
    syms = declared_symbols()
    assert "tce_w4a16_gemv" in syms and "tce_w8a8_matmul" in syms and "tce_attn_decode" in syms and len(syms) >= 20


def test_library_exports_every_declared_symbol(built_lib):
    L = C.CDLL(str(built_lib))
    for s in declared_symbols():
        assert hasattr(L, s), f"{s} declared in include/tce_b200.h but not exported by libtce_b200.so"


def test_python_binding_covers_header(built_lib):
    from tinychatengine_b200 import _lib

    assert sorted(_lib.SIGNATURES) == declared_symbols()
    _lib.lib()


def test_sass_is_hopper_native(built_lib):
    import subprocess

    sass = subprocess.run(["cuobjdump", "-sass", str(built_lib)], capture_output=True, text=True).stdout
    assert "sm_90a" in sass
    assert "UBLKCP" in sass, "TMA bulk copies missing from the W4A16 GEMV"
    assert "UTMALDG" in sass, "2-D TMA tensor copies missing (GEMV weight ring, wgmma GEMM operands)"
    assert "IMMA" in sass and "HMMA" in sass, "mma.sync paths missing (integer GEMV, attention)"
    assert "HGMMA" in sass and "IGMMA" in sass, "wgmma missing: the prefill / W8A8 GEMMs must run on the warpgroup tensor-core path"


def test_stream_k_partition_properties(tmp_path):
    """The GEMV's stream-K partition (csrc/kernels.h StreamK, shared by host and device code) compiled for the host: CTA ranges tile
    [0, U) exactly, are monotone, respect the cut granularity (whole stages / whole row tiles), and cta_of() inverts start()."""
    import subprocess

    src = tmp_path / "sk.cc"
    src.write_text(r"""
#include <cuda_runtime.h>
#include <stdio.h>
#include "kernels.h"
using tce::StreamK;
static int check(long long tiles, int NG, int nc, int aligned, int gran) {
    StreamK sk; sk.U = tiles * NG; sk.nc = nc; sk.NG = NG; sk.aligned = aligned; sk.T = (int)tiles; sk.gran = gran;
    if (sk.start(0) != 0 || sk.start(nc) != sk.U) return 1;
    for (int c = 0; c < nc; c++) {
        const long long a = sk.start(c), b = sk.start(c + 1);
        if (b < a) return 2;
        if (aligned ? (a % NG) : (a % gran)) return 3;
    }
    if (!aligned)
        for (long long u = 0; u < sk.U; u += (sk.U > 5000 ? 37 : 1)) {
            const int c = sk.cta_of(u);
            if (c < 0 || c >= nc || sk.start(c) > u || sk.start(c + 1) <= u) return 4;
        }
    return 0;
}
int main() {
    const long long tiles[] = {1, 3, 64, 256, 384, 1792, 8016};
    const int ngs[] = {1, 2, 16, 32, 86, 112}, ncs[] = {1, 7, 132, 148, 264, 296, 592};
    for (long long t : tiles) for (int ng : ngs) for (int nc : ncs) {
        const long long U = t * ng;
        for (int gran : {1, 16}) {
            if (U % gran) continue;
            int n = nc; if (n > U / gran) n = (int)(U / gran);
            if (int e = check(t, ng, n, 0, gran)) { printf("unaligned tiles=%lld NG=%d nc=%d gran=%d -> %d ", t, ng, n, gran, e); return 1; }
        }
        if (t >= nc) if (int e = check(t, ng, nc, 1, 1)) { printf("aligned tiles=%lld NG=%d nc=%d -> %d ", t, ng, nc, e); return 1; }
    }
    puts("ok");
    return 0;
}
""")
    exe = tmp_path / "sk"
    inc = ROOT / "tinychatengine_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-I/usr/local/cuda/include", f"-I{inc}", "-o", str(exe), str(src)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout


def test_slice_walk_properties(tmp_path):
    """The GEMV's unit walk (csrc/kernels.h SliceWalk, which every role of both GEMV kernels walks) compiled for the host.  With one slice it is
    the tile-major stream-K walk: the same CTA starts and pieces (rt = u / NG, gb = u % NG, up to the end of the tile or of the range).  With
    several slices the CTA ranges tile [0, T*NG), are monotone and start on (slice, tile) segment boundaries, the segments run slice-major,
    and locate() places every unit inside its segment."""
    import subprocess

    src = tmp_path / "walk.cc"
    src.write_text(r"""
#include <cuda_runtime.h>
#include <stdio.h>
#include "kernels.h"
using tce::SliceWalk;
using tce::StreamK;
static int check_one_slice(int T, int NG, int nc, int aligned, int gran) {
    const SliceWalk W{T, NG, NG, 1};
    StreamK sk; sk.U = (long long)T * NG; sk.nc = nc; sk.NG = NG; sk.aligned = aligned; sk.T = T; sk.gran = gran;
    for (int c = 0; c < nc; c++) {
        if (W.start(sk, c) != sk.start(c)) return 1;
        const int uend = W.start(sk, c + 1);
        for (int u = W.start(sk, c); u < uend;) {
            int s, rt, gb, seg0;
            W.locate(u, s, rt, gb, seg0);
            const int pe = uend < seg0 + W.len(s) ? uend : seg0 + W.len(s);
            const int rt_end = (u / NG + 1) * NG;
            if (s != 0 || rt != u / NG || gb != u % NG || pe != (uend < rt_end ? uend : rt_end)) return 2;
            u = pe;
        }
    }
    return 0;
}
static int check_slices(int T, int NG, int sl, int nc) {
    const int nsl = (NG + sl - 1) / sl;
    const SliceWalk W{T, NG, sl, nsl};
    const int U = T * NG;
    if (nc > T * nsl) nc = T * nsl;
    StreamK sk; sk.U = U; sk.nc = nc; sk.NG = NG; sk.T = T;
    // segments run slice-major: segment k = s*T + rt holds len(s) units, starting where segment k-1 ends
    if (W.seg_unit(0) != 0 || W.seg_unit((long long)T * nsl) != U) return 1;
    for (long long k = 0; k < (long long)T * nsl; k++)
        if (W.seg_unit(k + 1) - W.seg_unit(k) != W.len((int)(k / T))) return 2;
    if (W.start(sk, 0) != 0 || W.start(sk, nc) != U) return 3;
    for (int c = 0; c < nc; c++) {
        const int a = W.start(sk, c), b = W.start(sk, c + 1);
        if (b < a) return 4;
        int s, rt, gb, seg0;
        W.locate(a < U ? a : 0, s, rt, gb, seg0);
        if (nsl > 1 && a < U && seg0 != a) return 5;  // one slice keeps the stream-K cuts (checked above)
    }
    for (int u = 0; u < U; u += (U > 100000 ? 7 : 1)) {
        int s, rt, gb, seg0;
        W.locate(u, s, rt, gb, seg0);
        if (s < 0 || s >= nsl || rt < 0 || rt >= T || seg0 != W.seg_unit((long long)s * T + rt)) return 6;
        if (u < seg0 || u >= seg0 + W.len(s) || gb != s * sl + (u - seg0) || W.slice(u) != s) return 7;
    }
    return 0;
}
int main() {
    const int tiles[] = {1, 3, 256, 1792, 8016}, ngs[] = {8, 32, 86, 112}, ncs[] = {1, 7, 132, 264, 528};
    for (int t : tiles) for (int ng : ngs) for (int nc : ncs) {
        const long long U = (long long)t * ng;
        for (int gran : {1, 16}) {
            if (U % gran) continue;
            const int n = nc < U / gran ? nc : (int)(U / gran);
            if (int e = check_one_slice(t, ng, n, 0, gran)) { printf("one slice T=%d NG=%d nc=%d gran=%d -> %d ", t, ng, n, gran, e); return 1; }
        }
        if (t >= nc) if (int e = check_one_slice(t, ng, nc, 1, 1)) { printf("one slice aligned T=%d NG=%d nc=%d -> %d ", t, ng, nc, e); return 1; }
        for (int sl = 16; sl < ng; sl += 16)
            if (int e = check_slices(t, ng, sl, nc)) { printf("slices T=%d NG=%d sl=%d nc=%d -> %d ", t, ng, sl, nc, e); return 1; }
        if (int e = check_slices(t, ng, ng, nc)) { printf("slices T=%d NG=%d sl=NG nc=%d -> %d ", t, ng, nc, e); return 1; }
    }
    puts("ok");
    return 0;
}
""")
    exe = tmp_path / "walk"
    inc = ROOT / "tinychatengine_b200" / "csrc"
    subprocess.run(["g++", "-std=c++17", "-O2", "-I/usr/local/cuda/include", f"-I{inc}", "-o", str(exe), str(src)], check=True)
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout


@pytest.mark.skipif(torch.cuda.is_available(), reason="this checks the no-GPU behaviour")
def test_no_cpu_fallback(built_lib):
    from tinychatengine_b200 import _lib
    from tinychatengine_b200.runtime import Context

    L = _lib.lib()
    h = C.c_void_p()
    rc = L.tce_ctx_create(0, C.byref(h))
    assert rc == -3 and b"no CPU fallback" in L.tce_last_error()
    with pytest.raises(_lib.TceError):
        Context()


def test_zeros_width_matches_reference_rule(built_lib):
    from oracle import quant
    from tinychatengine_b200 import _lib, formats

    L = _lib.lib()
    for ic in (128, 1024, 1152, 4096, 5120, 11008, 13824, 14336):
        assert L.tce_zeros_width(ic, 128) == quant.calculate_zeros_width(ic, 128) == formats.zeros_width(ic, 128)
    assert L.tce_zeros_width(11008, 128) == 11 and L.tce_zeros_width(4096, 64) == 8


def test_header_is_plain_c(tmp_path):
    """include/tce_b200.h is the FFI contract: it must compile as C99 on its own (no C++ / CUDA / torch types in any signature)."""
    import subprocess

    src = tmp_path / "h.c"
    src.write_text('#include "tce_b200.h"\nint main(void) { return tce_version() < 0; }\n')
    r = subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-pedantic", "-fsyntax-only", f"-I{ROOT / 'include'}", str(src)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_product_never_touches_the_oracle(built_lib):
    """oracle/ is the checker: nothing under tinychatengine_b200/ may import, link or open it (the product path must fail without the CUDA
    library, not fall back to the CPU restatement), and bench.py may execute it only in the cpu_baseline / --impl reference legs."""
    import subprocess

    pkg = ROOT / "tinychatengine_b200"
    offenders = []
    for p in list(pkg.rglob("*.py")) + list(pkg.rglob("*.cu")) + list(pkg.rglob("*.cuh")) + list(pkg.rglob("*.h")) + list(pkg.rglob("Makefile")):
        if "build" in p.relative_to(pkg).parts[:1]:
            continue
        for n, line in enumerate(p.read_text(errors="replace").splitlines(), 1):
            code = line.split("//")[0].split("#")[0] if p.suffix != ".py" else line.split("#")[0]
            if re.search(r"\boracle\b|libtce_oracle|tce_oracle|orc_[a-z]", code) and "tests/cpp" not in line:
                offenders.append(f"{p.relative_to(ROOT)}:{n}: {line.strip()}")
    assert not offenders, "\n".join(offenders)
    # the shipped libraries do not link the oracle or any reference build
    for so in (pkg / "lib").glob("*.so"):
        needed = subprocess.run(["readelf", "-d", str(so)], capture_output=True, text=True).stdout
        assert "tce_oracle" not in needed and "tce_ref" not in needed, so
    # bench.py: every use of oracle/ sits inside the CPU-baseline class or the reference arm
    text = (ROOT / "bench.py").read_text()
    gpu_arm = text[text.index("def run_ours"):text.index("def main")]
    body = re.sub(r"cpu_baseline\([^\n]*", "", gpu_arm)
    assert "oracle" not in body and "capi" not in body
