"""CPU checks of the drop-in boundary: the C-ABI library loads and exports exactly the symbols
include/rcmarl.h declares (no compute without a GPU); the ctypes mirrors have the C layout."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    src = open(os.path.join(ROOT, "include", "rcmarl.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rcmarl_[a-z_0-9]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    from rcmarl import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__ as g
        g.build()
    lib = _lib.lib()
    declared = header_functions()
    bound = sorted(n for n, _, _ in _lib.SYMBOLS)
    assert declared == bound, (set(declared) ^ set(bound))
    for name in declared:
        assert hasattr(lib, name)
    assert b"sm_90a" in lib.rcmarl_version()
    assert lib.rcmarl_status_string(-2) == b"workspace too small"


def test_param_counts_and_workspace_query():
    from rcmarl import _lib
    lib = _lib.lib()
    assert lib.rcmarl_param_count(10, 1) == 661 == _lib.param_count(10, 1)      # critic, SURVEY 0
    assert lib.rcmarl_param_count(15, 1) == 761
    assert lib.rcmarl_param_count(10, 5) == 745
    assert lib.rcmarl_param_count(32, 1) == 1101 and lib.rcmarl_param_count(48, 1) == 1421   # C3
    assert lib.rcmarl_workspace_bytes(8, 761) >= 264 * 8 * 762 * 4 // 8         # two CTAs per SM on 132 SMs


def test_bad_arguments_are_rejected_without_a_device():
    from rcmarl import _lib
    lib = _lib.lib()
    assert lib.rcmarl_clip_mean(None, 4, 16, 16, 1, None, None) == -1
    assert lib.rcmarl_clip_mean(1, 4, 16, 16, 4, 1, None) == -1                 # H >= n
    assert lib.rcmarl_consensus_hidden(None, 1, None) == -1


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from rcmarl import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.RcmarlError):
        _lib.lib()


def test_struct_layouts_match_header_sizes(tmp_path):
    """sizeof() of every ABI struct as gcc sees include/rcmarl.h == the ctypes mirrors."""
    import shutil
    import subprocess
    from rcmarl import _lib as L
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    names = ["rcmarl_rows", "rcmarl_consensus_job", "rcmarl_value_job", "rcmarl_grad_job", "rcmarl_sgd_job",
             "rcmarl_adam_job", "rcmarl_team_job", "rcmarl_rollout_args"]
    mirrors = [L.Rows, L.ConsensusJob, L.ValueJob, L.GradJob, L.SgdJob, L.AdamJob, L.TeamJob, L.RolloutArgs]
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include "rcmarl.h"\nint main(){' +
                   "".join(f'printf("%zu\\n", sizeof({n}));' for n in names) + "return 0;}")
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    assert sizes == [ctypes.sizeof(m) for m in mirrors]


def test_product_tree_never_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under resilient-consensus-based-marl_b200/ may import or execute it."""
    prod = os.path.join(ROOT, "resilient-consensus-based-marl_b200")
    offenders = []
    for dirpath, _dirs, files in os.walk(prod):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f), errors="replace").read()
                if re.search(r"^\s*(from|import)\s+oracle\b|rpbcac_oracle|tf_facade", txt, re.M):
                    offenders.append(os.path.join(dirpath, f))
    assert not offenders, offenders
