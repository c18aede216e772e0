"""Host side of the deterministic mode (torch.use_deterministic_algorithms -> ymp_set_deterministic): the C switch, the
rule that maps torch's flags to it, the CUDA-graph key of TrainEngine.train_step, and the launcher's --ymp-pre hook
that turns the flag on for an unmodified script.  The kernels are checked in test_deterministic_gpu.py."""
import os
import subprocess
import sys
import textwrap

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "youku-mplug_b200")


def test_set_deterministic_round_trips_previous_value():
    from ymp import lib as L
    prev = L.lib.ymp_set_deterministic(0)
    try:
        assert L.lib.ymp_set_deterministic(1) == 0
        assert L.lib.ymp_set_deterministic(1) == 1
        assert L.lib.ymp_set_deterministic(7) == 1       # any non-zero value means on
        assert L.lib.ymp_set_deterministic(0) == 1
        assert L.lib.ymp_set_deterministic(0) == 0
    finally:
        L.lib.ymp_set_deterministic(prev)


def test_workspace_sizes_are_zero_with_the_mode_off():
    from ymp import lib as L
    prev = L.lib.ymp_set_deterministic(0)
    try:
        a = L.ColsumArgs()
        a.R, a.C, a.ld = 4096, 768, 768
        assert L._colsum_ws_size(L.C.byref(a)) == 0
        assert L._sumsq_ws_size(1 << 20) == 0
        L.lib.ymp_set_deterministic(1)
        assert L._colsum_ws_size(L.C.byref(a)) > 0 and L._colsum_ws_size(L.C.byref(a)) % 16 == 0
        assert L._sumsq_ws_size(1 << 20) > 0
    finally:
        L.lib.ymp_set_deterministic(prev)


def test_mode_rule_is_a_pure_function_of_torchs_flags():
    from ymp import lib as L
    assert L.deterministic_mode(False, False) == 0
    assert L.deterministic_mode(True, False) == 1
    assert L.deterministic_mode(True, True) == 1     # enabled with warn_only counts as on
    assert L.deterministic_mode(False, True) == 0    # use_deterministic_algorithms(False, warn_only=True): off
    assert [L.deterministic_mode(True, False) for _ in range(3)] == [1, 1, 1]


def test_sync_follows_use_deterministic_algorithms():
    from ymp import lib as L
    prev_c = L.lib.ymp_set_deterministic(0)
    prev_t, prev_w = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    try:
        for on, warn in ((True, False), (False, False), (True, True), (False, True), (False, False)):
            torch.use_deterministic_algorithms(on, warn_only=warn)
            assert torch.is_deterministic_algorithms_warn_only_enabled() == warn
            assert L.sync_deterministic() == int(on)
            assert L.lib.ymp_set_deterministic(int(on)) == int(on)    # the library holds the same value
    finally:
        torch.use_deterministic_algorithms(prev_t, warn_only=prev_w)
        L.lib.ymp_set_deterministic(prev_c)


def test_train_step_graph_key_changes_with_the_mode():
    from ymp import train
    prev_t, prev_w = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    x = torch.zeros(2, 3)
    try:
        torch.use_deterministic_algorithms(False)
        off = train.graph_key([x, None])
        torch.use_deterministic_algorithms(True)
        on = train.graph_key([x, None])
        torch.use_deterministic_algorithms(True, warn_only=True)
        warn = train.graph_key([x, None])
        torch.use_deterministic_algorithms(False, warn_only=True)
        warn_off = train.graph_key([x, None])
    finally:
        torch.use_deterministic_algorithms(prev_t, warn_only=prev_w)
    assert off != on and on == warn and warn_off == off
    assert off[1:] == on[1:]                     # the input signature is the same; only the mode differs
    assert train.graph_key([torch.ones(2, 3)]) != train.graph_key([torch.ones(2, 4)])


def test_ymp_pre_file_enables_the_flag_before_the_script(tmp_path):
    pre = tmp_path / "deterministic.py"
    pre.write_text("import torch\ntorch.use_deterministic_algorithms(True)\n")
    script = tmp_path / "script.py"
    script.write_text(textwrap.dedent("""
        import torch
        from ymp import lib
        print("FLAG", torch.are_deterministic_algorithms_enabled(), lib.sync_deterministic())
    """))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([PKG, ROOT]))
    r = subprocess.run([sys.executable, os.path.join(PKG, "launch.py"), "--ymp-pre", str(pre), "--ymp-standalone", str(script)],
                       capture_output=True, text=True, env=env, cwd=str(tmp_path), timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert "FLAG True 1" in r.stdout, r.stdout[-2000:]
