#!/usr/bin/env python
"""Run one of the reference's scripts UNMODIFIED on the H100 `models` package.

    python youku-mplug_b200/launch.py /path/to/Youku-mPLUG/run_pretrain_distributed_gpt3.py \
        --config configs/pretrain/gpt3_1.3B/pretrain_gpt3_freezeGPT_youku_v0.yaml --output_dir out \
        --enable_deepspeed --bf16
    python -m torch.distributed.run --nproc-per-node 8 youku-mplug_b200/launch.py <script> <args ...>

What it does before handing control to the script (runpy, `__main__`):
  1. puts this directory first on sys.path and imports the H100 `models` package, then appends the reference's own
     `models/` directory to `models.__path__`: `models.distributed_gpt3`, `models.modeling_distributed_gpt3`,
     `models.vision_transformer`, `models.distributed_utils`, `models.model_pretrain_gpt` resolve HERE, every other
     submodule the scripts' imports pull in (`models.tokenization_bert` via `dataset/grounding_dataset.py:28`,
     ...) still resolves in the reference.  (A plain `PYTHONPATH=` does not work: Python puts the script's own
     directory at sys.path[0], ahead of PYTHONPATH.)
  2. puts the reference checkout (the script's repository root) next on sys.path for `utils`, `dataset`, `optim`,
     `scheduler`;
  3. appends `compat/` (stand-ins for deepspeed / megatron_util / ruamel.yaml / timm / addict / sh / tensorboardX /
     decord, see compat/README.md) to the END of sys.path so that really installed packages win - except
     `deepspeed`, whose `initialize()` must return the H100 engine (set YMP_KEEP_DEEPSPEED=1 to keep a real one);
  4. restores three private helpers transformers 5.x removed and the reference's BERT tokenizer imports
     (models/tokenization_bert.py:23);
  5. optional `--ymp-pre FILE`: a Python file executed first (site-specific hooks, e.g. registering a dataset).
"""
import importlib.util
import os
import runpy
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
COMPAT = os.path.join(HERE, "compat")


def _reference_root(script):
    d = os.path.dirname(os.path.abspath(script))
    while d != os.path.dirname(d):
        if os.path.isdir(os.path.join(d, "models")) and os.path.isfile(os.path.join(d, "utils.py")):
            return d
        d = os.path.dirname(d)
    raise SystemExit(f"launch.py: cannot find the reference checkout (a directory with models/ and utils.py) above {script}")


def prepare(script, need_reference=True):
    ref = _reference_root(script) if need_reference else None
    for p in (HERE, ref):
        while p in sys.path:
            sys.path.remove(p)
    if ref:
        sys.path.insert(0, ref)
    sys.path.insert(0, HERE)
    if COMPAT not in sys.path:
        sys.path.append(COMPAT)
    if os.environ.get("YMP_KEEP_DEEPSPEED", "0") != "1":
        spec = importlib.util.spec_from_file_location("deepspeed", os.path.join(COMPAT, "deepspeed", "__init__.py"),
                                                      submodule_search_locations=[os.path.join(COMPAT, "deepspeed")])
        mod = importlib.util.module_from_spec(spec)
        sys.modules["deepspeed"] = mod
        spec.loader.exec_module(mod)
    import transformers  # noqa: F401  (before any timm stand-in is importable: its availability probe inspects timm)
    import transformers.tokenization_utils as tu
    import unicodedata

    def _is_whitespace(char):
        return char in (" ", "\t", "\n", "\r") or unicodedata.category(char) == "Zs"

    def _is_control(char):
        if char in ("\t", "\n", "\r"):
            return False
        return unicodedata.category(char).startswith("C")

    def _is_punctuation(char):
        cp = ord(char)
        if (33 <= cp <= 47) or (58 <= cp <= 64) or (91 <= cp <= 96) or (123 <= cp <= 126):
            return True
        return unicodedata.category(char).startswith("P")

    for name, fn in (("_is_whitespace", _is_whitespace), ("_is_control", _is_control), ("_is_punctuation", _is_punctuation)):
        if not hasattr(tu, name):
            setattr(tu, name, fn)
    import models  # the H100 package (HERE is first on sys.path)
    assert os.path.dirname(os.path.abspath(models.__file__)) == os.path.join(HERE, "models"), models.__file__
    if ref:
        ref_models = os.path.join(ref, "models")
        if ref_models not in models.__path__:
            models.__path__.append(ref_models)
    return ref


def main(argv):
    pre, need_ref = None, True
    while argv and argv[0].startswith("--ymp-"):
        if argv[0] == "--ymp-pre" and len(argv) >= 2:
            pre, argv = argv[1], argv[2:]
        elif argv[0] == "--ymp-standalone":      # a script that lives outside a reference checkout (own training loops)
            need_ref, argv = False, argv[1:]
        else:
            raise SystemExit(f"launch.py: unknown option {argv[0]}")
    if not argv:
        raise SystemExit(__doc__)
    script, args = argv[0], argv[1:]
    prepare(script, need_ref)
    if pre:
        runpy.run_path(pre, run_name="__ymp_pre__")
    sys.argv = [script] + args
    runpy.run_path(script, run_name="__main__")


if __name__ == "__main__":
    main(sys.argv[1:])
