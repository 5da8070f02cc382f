"""Alias package: `import dalm...` resolves to dalm_b200's drop-in modules, so code written against the reference's
import paths (dalm.models.*, dalm.training.*, dalm.cli, dalm.utils) runs unchanged on the H100 build.

`dalm.X` IS `dalm_b200.X` (the same module object, executed once): the finder hands the import machinery a spec whose
loader returns the already-imported real module from `create_module` and does nothing in `exec_module`, so module
globals (mode switches, stream caches) and classes (isinstance checks in save_model_hook) exist exactly once."""
import importlib
import importlib.abc
import importlib.util
import sys

import dalm_b200
from dalm_b200 import __version__  # noqa: F401

_ALIASES = [
    "cli", "utils", "models", "models.rag_e2e_base_model", "models.retriever_only_base_model", "training",
    "training.utils", "training.utils.train_utils", "training.utils.rag_e2e_dataloader_utils",
    "training.utils.retriever_only_dataloader_utils", "training.rag_e2e", "training.rag_e2e.train_rage2e",
    "training.retriever_only", "training.retriever_only.train_retriever_only",
    "eval", "eval.utils", "eval.eval_results", "eval.eval_retriever_only", "eval.eval_rag",
]


class _AliasLoader(importlib.abc.Loader):
    def __init__(self, real_name: str):
        self.real_name = real_name

    def create_module(self, spec):
        real = importlib.import_module(self.real_name)       # the one and only module object
        self._real_spec = real.__spec__
        return real

    def exec_module(self, module):                           # already executed under its real name
        module.__spec__ = self._real_spec                    # the machinery stamped the alias spec on it: put the real one back
        return None


class _LazyAlias(importlib.abc.MetaPathFinder):
    """meta-path finder mapping dalm.X -> dalm_b200.X on first import"""

    @staticmethod
    def find_spec(name, path=None, target=None):
        if not name.startswith("dalm.") or name[5:] not in _ALIASES:
            return None
        real_name = "dalm_b200." + name[5:]
        real = importlib.import_module(real_name)
        spec = importlib.util.spec_from_loader(name, _AliasLoader(real_name), is_package=hasattr(real, "__path__"))
        if spec is not None and hasattr(real, "__path__"):
            spec.submodule_search_locations = list(real.__path__)
        return spec


sys.meta_path.insert(0, _LazyAlias)
