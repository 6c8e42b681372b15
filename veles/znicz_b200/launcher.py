"""Command line launcher (the ``veles`` script equivalent; SURVEY §3.1 call stack).

    python -m veles.znicz_b200 [options] <workflow.py | module> [config.py] [root.a.b=value ...]

A workflow file exposes ``run(load, main)`` exactly like the reference samples
(/root/reference/samples/Wine/wine.py:176-181): ``load(WorkflowClass, **kwargs)`` builds
the workflow (or restores it from ``--snapshot``) and returns ``(workflow, restored)``;
``main(**kwargs)`` initialises it on the selected device and runs it.

Under ``torchrun`` every rank executes the same command; ``StandardWorkflow.initialize``
picks the data-parallel context up from the environment (one process per GPU).
"""
from __future__ import annotations

import argparse
import importlib
import importlib.util
import json
import logging
import os
import sys
import time

import numpy

from .core import genetics, prng
from .core.config import root
from .core.workflow import DummyLauncher


class Launcher(DummyLauncher):
    """Owns the run mode, the device choice and the life cycle of one workflow."""

    def __init__(self, backend="auto", testing=False, snapshot=None, result_file=None,
                 dry_run=None, stealth=False, **kwargs):
        super().__init__(mode=kwargs.pop("mode", "standalone"), testing=testing)
        self.backend = backend
        self.snapshot = snapshot
        self.result_file = result_file
        self.dry_run = dry_run
        self.restored = False
        self.start_time = None
        self.run_time = 0.0

    # -- load / main passed to the workflow module --------------------------------------------
    @staticmethod
    def resolve_snapshot(spec):
        """``latest`` / ``latest:<prefix>`` -> the newest snapshot of the snapshot directory
        (the ``<prefix>_current.lnk`` symlink when it exists), None when there is none yet - what
        a job restarted by ``torchrun --max-restarts`` after a rank failure resumes from."""
        if not spec or not str(spec).startswith("latest"):
            return spec
        prefix = str(spec).partition(":")[2]
        directory = str(root.common.dirs.snapshots)
        if not os.path.isdir(directory):
            return None
        names = [n for n in os.listdir(directory) if ".pickle" in n and ".tmp." not in n and
                 (not prefix or n.startswith(prefix + "_"))]
        link = os.path.join(directory, "%s_current.lnk" % prefix) if prefix else None
        if link and os.path.exists(link):
            return link
        if not names:
            return None
        return max((os.path.join(directory, n) for n in names), key=os.path.getmtime)

    def load(self, workflow_class, **kwargs):
        self.snapshot = self.resolve_snapshot(self.snapshot)
        if self.snapshot:
            from .core.snapshotter import SnapshotterToFile
            wf = SnapshotterToFile.import_file(self.snapshot)
            if not isinstance(wf, workflow_class):
                logging.getLogger("Launcher").warning(
                    "snapshot holds %s, expected %s", type(wf).__name__,
                    workflow_class.__name__)
            wf.workflow = self
            self.restored = True
        else:
            wf = workflow_class(self, **kwargs)
        self.workflow = wf
        if self.result_file:
            wf.result_file = self.result_file
        return wf, self.restored

    def main(self, **kwargs):
        wf = self.workflow
        if wf is None:
            raise RuntimeError("main() called before load()")
        if self.dry_run == "load":
            return wf
        kwargs.setdefault("device", self.backend)
        if self.restored:
            kwargs.setdefault("snapshot", True)
        self.start_time = time.time()
        wf.initialize(**kwargs)
        if self.dry_run == "init":
            return wf
        wf.run()
        self.run_time = time.time() - self.start_time
        wf.print_stats()
        return wf


def _set_by_path(path, value):
    parts = path.split(".")
    if parts[0] == "root":
        parts = parts[1:]
    node = root
    for p in parts[:-1]:
        node = getattr(node, p)
    setattr(node, parts[-1], value)


def _parse_value(text):
    try:
        return json.loads(text)
    except ValueError:
        pass
    try:
        return eval(text, {"numpy": numpy, "Range": genetics.Range})  # noqa: S307 (own CLI)
    except Exception:
        return text


def import_workflow_module(spec):
    if os.path.exists(spec):
        name = "znicz_workflow_" + os.path.splitext(os.path.basename(spec))[0]
        s = importlib.util.spec_from_file_location(name, spec)
        mod = importlib.util.module_from_spec(s)
        sys.modules[name] = mod
        s.loader.exec_module(mod)
        return mod
    if "." not in spec:
        spec = "veles.znicz_b200.models." + spec
    return importlib.import_module(spec)


def apply_config_file(path):
    from . import compat  # noqa: F401  (lets reference configs ``from veles.config import root``)
    with open(path) as f:
        code = compile(f.read(), path, "exec")
    exec(code, {"__file__": path, "__name__": "__znicz_config__", "root": root,
                "Range": genetics.Range})


def build_parser():
    p = argparse.ArgumentParser(
        prog="python -m veles.znicz_b200",
        description="Run a Znicz workflow on H100 (or the numpy backend).")
    p.add_argument("workflow", help="workflow .py file, dotted module or sample name "
                                    "(wine, mnist, cifar, ...)")
    p.add_argument("config", nargs="?", default=None,
                   help="config .py file (use - for none)")
    p.add_argument("overrides", nargs="*", help="root.path.to.key=value assignments")
    p.add_argument("-b", "--backend", default=None, choices=("auto", "cuda", "numpy"))
    p.add_argument("-s", "--snapshot", default=None,
                   help="resume from this snapshot file; 'latest[:prefix]' = the newest one in "
                        "root.common.dirs.snapshots, a fresh start when there is none (restart "
                        "after a rank failure: torchrun --max-restarts N ... --snapshot latest)")
    p.add_argument("--test", action="store_true", help="testing mode (forward only)")
    p.add_argument("--result-file", default=None, help="write gathered metrics as JSON")
    p.add_argument("--dry-run", default=None, choices=("load", "init"))
    p.add_argument("--seed", type=int, default=None, help="seed of both host generators")
    p.add_argument("--optimize", default=None, metavar="POP[:GEN]",
                   help="genetic search over Range(...) markers of the config")
    p.add_argument("--dump-config", action="store_true")
    p.add_argument("--no-graphs", action="store_true", help="disable CUDA-graph segments")
    p.add_argument("--compute", default=None, choices=("fp32", "bf16", "fp8"))
    p.add_argument("-v", "--verbosity", default="info",
                   choices=("debug", "info", "warning", "error"))
    return p


def _fitness(wf):
    res = wf.gather_results()
    for key in ("EvaluationFitness", "fitness"):
        if key in res:
            return float(res[key])
    dec = getattr(wf, "decision", None)
    if dec is not None:
        pt = getattr(dec, "best_n_err_pt", None)
        if pt is not None and pt[1] is not None:
            return 100.0 - float(pt[1])
        mse = getattr(dec, "best_mse", None) or getattr(dec, "min_validation_mse", None)
        if mse is not None:
            return -float(mse if numpy.isscalar(mse) else mse[1])
    raise RuntimeError("the workflow does not expose a fitness metric")


def run_once(args, module):
    launcher = Launcher(backend=args.backend or root.common.engine.get("backend", "auto"),
                        testing=args.test, snapshot=args.snapshot,
                        result_file=args.result_file, dry_run=args.dry_run)
    module.run(launcher.load, launcher.main)
    return launcher


def main(argv=None):
    args = build_parser().parse_args(argv)
    logging.basicConfig(level=getattr(logging, args.verbosity.upper()),
                        format="%(asctime)s %(levelname)s %(name)s: %(message)s")
    # positional "config" may really be the first override
    if args.config and "=" in args.config and not os.path.exists(args.config):
        args.overrides.insert(0, args.config)
        args.config = None
    if args.seed is not None:
        prng.get(1).seed(args.seed)
        prng.get(2).seed(args.seed + 1)
    module = import_workflow_module(args.workflow)    # defaults are set at import time
    if args.config and args.config != "-":
        apply_config_file(args.config)
    for ov in args.overrides:
        k, _, v = ov.partition("=")
        _set_by_path(k.strip(), _parse_value(v.strip()))
    if args.no_graphs:
        root.common.engine.graphs = False
    if args.compute:
        root.common.engine.compute_type = args.compute
    if args.dump_config:
        root.print_()
    if args.optimize:
        pop, _, gen = args.optimize.partition(":")
        markers = genetics.process_config(root)
        rank = int(os.environ.get("RANK", "0"))

        def evaluate(values):
            genetics.apply_values(root, markers, values)
            old = root.common.disable.snapshotting
            root.common.disable.snapshotting = True
            try:
                launcher = run_once(args, module)
            finally:
                root.common.disable.snapshotting = old
            return _fitness(launcher.workflow)
        opt = genetics.GeneticsOptimizer(
            markers, evaluate, population_size=int(pop), generations=int(gen or 3),
            seed=args.seed or 1, log=logging.getLogger("Genetics").info)
        best, fit = opt.run()
        if rank == 0:
            print(json.dumps({"best_fitness": fit,
                              "best": {".".join(map(str, m[0])): v
                                       for m, v in zip(markers, best)}}, default=str))
        return 0
    genetics.fix_config(root)
    launcher = run_once(args, module)
    wf = launcher.workflow
    if wf is not None and args.dry_run is None and int(os.environ.get("RANK", "0")) == 0:
        print(json.dumps(wf.gather_results(), default=str))
    return 0
