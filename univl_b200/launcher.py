"""Compat launcher: run an UNMODIFIED microsoft/UniVL driver on univl_b200 (SURVEY.md §8f#4).

    python -m torch.distributed.run --nproc_per_node=8 -m univl_b200.launcher \
        /path/to/UniVL/main_task_retrieval.py --do_train --bert_model /path/to/bert-base-uncased ...

What it does before handing over to the driver (`runpy.run_path(..., run_name="__main__")`):
  * puts the UniVL checkout first on sys.path (the drivers import `metrics`, `util`, `dataloaders.*` from it);
  * shadows the reference package `modules` with `univl_b200.modules` (modeling, module_*, until_*, optimization,
    file_utils) and loads the checkout's own `modules/tokenization.py` and `modules/beam.py` (CPU string / search code,
    out of scope here) under their reference names;
  * stubs import-time dependencies that are absent on the target machines and unused on the hot path: `boto3` /
    `botocore` (modules/file_utils.py:20-21) and `nlgeval` (main_task_caption.py:12 — caption *metrics* only; the stub
    raises if a metric is actually requested);
  * restores the numpy aliases removed in numpy >= 1.24 that the dataloaders use (`np.float`, e.g.
    dataloaders/dataloader_youcook_retrieval.py:139);
  * maps torchrun's `--local-rank` / LOCAL_RANK to the `--local_rank` argument the drivers parse
    (main_task_retrieval.py:83), and fills MASTER_ADDR / MASTER_PORT / RANK / WORLD_SIZE for a single-process run so
    the import-time `torch.distributed.init_process_group(backend="nccl")` (main_task_retrieval.py:23) succeeds.
Nothing of the reference checkout is modified or copied.
"""
import importlib
import importlib.util
import os
import runpy
import sys
import types

_SHADOWED = ("modeling", "module_bert", "module_visual", "module_cross", "module_decoder", "until_module",
             "until_config", "optimization", "file_utils")


def install_stubs():
    for name in ("boto3", "botocore", "botocore.exceptions"):
        if name not in sys.modules:
            try:
                importlib.import_module(name)
            except ImportError:
                sys.modules[name] = types.ModuleType(name)
    exc = sys.modules["botocore.exceptions"]
    if not hasattr(exc, "ClientError"):
        exc.ClientError = type("ClientError", (Exception,), {})
    if not hasattr(sys.modules["botocore"], "exceptions"):
        sys.modules["botocore"].exceptions = exc
    try:
        importlib.import_module("nlgeval")
    except ImportError:
        stub = types.ModuleType("nlgeval")

        class NLGEval(object):  # noqa: D401 — same constructor signature as nlgeval.NLGEval
            def __init__(self, *a, **k):
                pass

            def compute_metrics(self, *a, **k):
                raise RuntimeError("nlgeval is not installed: caption metrics (BLEU/METEOR/ROUGE/CIDEr) are outside "
                                   "univl_b200; install nlg-eval to score captions")
        stub.NLGEval = NLGEval
        sys.modules["nlgeval"] = stub


def install_numpy_aliases():
    import numpy as np
    for alias, target in (("float", float), ("int", int), ("bool", bool), ("object", object)):
        if not hasattr(np, alias):
            setattr(np, alias, target)


def install_shadow(checkout):
    """`from modules.X import ...` resolves to univl_b200.modules.X for the hot-path modules and to the checkout's own
    file for tokenization / beam.  Under UNIVL_DECODE_CACHE=prefix, `modules.beam` is univl_b200.modules.beam, whose
    Beam keeps its hypotheses on the host."""
    from .caption import decode_cache_mode
    checkout = os.path.abspath(checkout)
    if checkout not in sys.path:
        sys.path.insert(0, checkout)
    pkg = importlib.import_module("univl_b200.modules")
    sys.modules["modules"] = pkg
    shadowed = _SHADOWED + (("beam",) if decode_cache_mode() == "prefix" else ())
    for name in shadowed:
        sys.modules["modules." + name] = importlib.import_module("univl_b200.modules." + name)
    for name in ("tokenization", "beam"):
        if name in shadowed:
            setattr(pkg, name, sys.modules["modules." + name])
            continue
        path = os.path.join(checkout, "modules", name + ".py")
        if not os.path.exists(path):
            continue
        spec = importlib.util.spec_from_file_location("modules." + name, path)
        mod = importlib.util.module_from_spec(spec)
        mod.__package__ = "modules"
        sys.modules["modules." + name] = mod
        spec.loader.exec_module(mod)
        setattr(pkg, name, mod)
    return checkout


def fix_rank_args(argv):
    """torch >= 2 launchers pass --local-rank (or only LOCAL_RANK); the drivers parse --local_rank."""
    out, seen = [], False
    for a in argv:
        if a.startswith("--local-rank"):
            a = "--local_rank" + a[len("--local-rank"):]
        if a.startswith("--local_rank"):
            seen = True
        out.append(a)
    if not seen and "LOCAL_RANK" in os.environ:
        out += ["--local_rank", os.environ["LOCAL_RANK"]]
    return out


def single_process_env():
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29531")
    os.environ.setdefault("RANK", "0")
    os.environ.setdefault("WORLD_SIZE", "1")
    os.environ.setdefault("LOCAL_RANK", "0")


def prepare(driver_path):
    install_stubs()
    install_numpy_aliases()
    single_process_env()
    return install_shadow(os.path.dirname(os.path.abspath(driver_path)))


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv or argv[0] in ("-h", "--help"):
        print(__doc__)
        return 0
    driver = argv[0]
    prepare(driver)
    sys.argv = [driver] + fix_rank_args(argv[1:])
    runpy.run_path(driver, run_name="__main__")
    return 0


if __name__ == "__main__":
    sys.exit(main())
