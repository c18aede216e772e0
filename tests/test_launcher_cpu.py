"""The compat/ stand-ins the launcher (youku-mplug_b200/launch.py) installs for the reference's scripts: the YAML
loader must read YAML 1.2 floats as the scripts expect.  The script-level run through launch.py is
tests/test_launcher_gpu.py."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_compat_yaml_reads_yaml12_floats():
    sys.path.append(os.path.join(ROOT, "youku-mplug_b200", "compat"))
    try:
        import importlib
        y = importlib.import_module("ruamel.yaml")
        d = y.load("a: 1e-4\nb: 1e-6\nc: [0.9, 0.999]\nd: 3\ne: {x: 2e-5,}\nf: text\n", Loader=y.Loader)
        assert d == {"a": 1e-4, "b": 1e-6, "c": [0.9, 0.999], "d": 3, "e": {"x": 2e-5}, "f": "text"}
        assert isinstance(d["a"], float) and isinstance(d["d"], int)
    finally:
        sys.path.remove(os.path.join(ROOT, "youku-mplug_b200", "compat"))
        for k in [k for k in sys.modules if k == "ruamel" or k.startswith("ruamel.")]:
            del sys.modules[k]
