"""C-ABI contract (no GPU needed): libevcplm.so loads, exports every function include/evcplm.h declares, and the
ctypes binding (evcouplings_b200/_lib.py) covers exactly that set.  No compute entry point is called."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "evcplm.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)          # drop comments
    return set(re.findall(r"\b(evc_[a-z0-9_]+)\s*\(", text))


def test_header_binding_and_library_agree():
    from evcouplings_b200 import _lib
    declared = _declared()
    assert len(declared) >= 25
    assert declared == set(_lib.PROTOTYPES), (declared ^ set(_lib.PROTOTYPES))
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in sorted(declared):
        assert hasattr(lib, name), "libevcplm.so does not export " + name
    bound = _lib.load()
    assert bound.evc_abi_version() == _lib.ABI_VERSION == 2


def test_library_reports_errors_without_device():
    """argument validation and the error channel work without touching a GPU"""
    from evcouplings_b200 import _lib
    lib = _lib.load()
    assert lib.evc_plm_num_params(None) == -1
    assert lib.evc_hamming_num_tiles(300) == 6 and lib.evc_hamming_plane_words(300, 40) == 5 * 2 * 300
    rc = lib.evc_plm_set_backward(None, 1)
    assert rc != 0 and b"null handle" in lib.evc_last_error()
    rc = lib.evc_hamming_counts(None, 0, 0, 0, 0, None)
    assert rc != 0 and lib.evc_last_error()
    rc = lib.evc_plm_copy_stage(None, 0, None, 0)
    assert rc != 0 and b"evc_plm_copy_stage: null pointer" in lib.evc_last_error()


def test_stage_constants_match_the_binding():
    """the EVC_STAGE_* defines of include/evcplm.h are the numbers _lib.STAGE passes to evc_plm_copy_stage"""
    from evcouplings_b200 import _lib
    text = open(os.path.join(ROOT, "include", "evcplm.h")).read()
    defines = {k: int(v) for k, v in re.findall(r"#define EVC_STAGE_(\w+) (\d+)", text)}
    assert defines == {k.upper(): v for k, v in _lib.STAGE.items()}
    assert sorted(defines.values()) == list(range(len(defines)))


def test_create_validates_code_range_before_touching_a_device():
    """ADVICE r1 (medium): a code >= q (q + 1 with the ignored gap) must be rejected, not used as a row index."""
    import numpy as np
    from evcouplings_b200 import _lib
    lib = _lib.load()
    w = np.ones(4, dtype=np.float32)
    h = ctypes.c_void_p()
    for q, gap, bad in ((21, -1, 21), (20, 20, 21), (4, -1, 200)):
        codes = np.zeros((4, 3), dtype=np.uint8)
        codes[2, 1] = bad
        rc = lib.evc_plm_create(ctypes.byref(h), codes.ctypes.data_as(ctypes.c_void_p), 4, 3, q, gap,
                                w.ctypes.data_as(ctypes.c_void_p), 0)
        assert rc != 0 and b"out of range" in lib.evc_last_error(), lib.evc_last_error()


def test_compiled_a2m_reader_matches_python_reader(tmp_path):
    """f4: csrc/a2m_reader.cu against the pure-Python line loop: wrapped records, CRLF, blank lines, text before the
    first header, lower-case inserts and '.'; error classes for empty / ragged / zero-length input."""
    import numpy as np
    import pytest
    from evcouplings_b200 import msa
    text = ("junk before the first record\n>seqA/5-14 some description\r\nACDEF\r\nghik.\n\n>seqB\n"
            "AC-EFGH\nIK.\n>seqC\nacdefGHIK-\n")
    p = tmp_path / "a.a2m"
    p.write_bytes(text.encode())
    ids, raw = msa.read_fasta_matrix(str(p))
    ids_py, raw_py = msa.read_fasta_matrix_py(str(p))
    assert ids == ids_py == ["seqA/5-14 some description", "seqB", "seqC"]
    assert raw.shape == (3, 10) and np.array_equal(raw, raw_py)
    ali = msa.load_alignment(str(p), focus="seqA")
    assert ali.region_start == 5 and ali.target_seq == "ACDEF" and ali.codes.shape == (3, 5)
    for bad, msg in ((b"", "no sequences"), (b">a\nAC\n>b\nACD\n", "ragged"), (b">a\n>b\n", "zero-length")):
        q = tmp_path / "bad.a2m"
        q.write_bytes(bad)
        with pytest.raises(msa.AlignmentError, match=msg):
            msa.read_fasta_matrix(str(q))
        with pytest.raises(msa.AlignmentError, match=msg):
            msa.read_fasta_matrix_py(str(q))


def test_header_is_plain_c(tmp_path):
    """include/evcplm.h is the drop-in boundary: it must compile as C (C99, -pedantic), no C++ / torch types."""
    import subprocess
    src = tmp_path / "hdr.c"
    src.write_text('#include "evcplm.h"\n'
                   'int main(void) { evc_fit_params_t p; evc_fit_result_t r; (void)r; evc_fit_default_params(&p);\n'
                   '  return evc_abi_version() == EVCPLM_ABI_VERSION ? 0 : 1; }\n')
    p = subprocess.run(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-fsyntax-only",
                        "-I", os.path.join(ROOT, "include"), str(src)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr


def test_c_program_links_and_calls_the_library(tmp_path):
    """A plain C host (what a non-Python binding of the reference's plmc call site would be) links against
    libevcplm.so and uses the device-independent entry points."""
    import subprocess
    from evcouplings_b200 import _lib
    src = tmp_path / "host.c"
    src.write_text(r'''
#include <stdio.h>
#include "evcplm.h"
int main(void) {
    evc_fit_params_t p;
    evc_fit_default_params(&p);
    int rc = evc_plm_set_backward(NULL, 1);
    printf("%d %lld %lld %d %d %s\n", evc_abi_version(), (long long)evc_hamming_num_tiles(300),
           (long long)evc_hamming_plane_words(300, 40), (int)p.m, rc, evc_last_error());
    return 0;
}
''')
    exe = tmp_path / "host"
    libdir = os.path.dirname(_lib.LIB_PATH)
    c = subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe), "-L", libdir,
                        "-levcplm", "-Wl,-rpath," + libdir], capture_output=True, text=True)
    assert c.returncode == 0, c.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = r.stdout.split(None, 5)
    assert out[:5] == [str(_lib.ABI_VERSION), "6", "3000", "6", "1"] and "null handle" in out[5]


def test_shipped_library_is_hopper_native():
    """SASS evidence that the tensor-core path is built for Hopper: wgmma -> HGMMA, TMA tensor loads -> UTMALDG, bulk
    copies -> UBLKCP, the producer / consumer register split -> USETMAXREG; no legacy HMMA path in the GEMM kernels.
    Skipped where cuobjdump is not installed."""
    import shutil
    import subprocess
    import pytest
    from evcouplings_b200 import _lib
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe):
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], capture_output=True, text=True, timeout=600).stdout
    assert "sm_90a" in sass
    for mnemonic in ("HGMMA", "UTMALDG", "UBLKCP", "USETMAXREG"):
        assert mnemonic in sass, mnemonic
    gemm = sass[sass.index("tc_gemm_kernel"):]
    gemm = gemm[:gemm.index("Function :", 20)] if "Function :" in gemm[20:] else gemm
    assert "HGMMA" in gemm and " HMMA" not in gemm
