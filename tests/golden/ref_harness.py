"""
Import the (Python) reference EVcouplings: from the checkout named by the environment variable EVC_REFERENCE, or
from the git-ignored install baseline/_ref (scripts/install_reference.sh).

The reference's optional plotting / batch dependencies are absent here
(ruamel.yaml, matplotlib, seaborn, bokeh, billiard, Bio); none of them is on
the couplings path, so they are shimmed (SURVEY.md Appendix B).  Used by
tests/golden/make_golden.py (golden-vector generation) and by the boundary
tests, which skip when the reference is absent.
"""
import importlib.abc
import importlib.machinery
import os
import sys
import types
import warnings
from unittest import mock

_REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_CANDIDATES = tuple(c for c in (os.environ.get("EVC_REFERENCE"), os.path.join(_REPO, "baseline", "_ref")) if c)
REFERENCE_ROOT = next((c for c in _CANDIDATES if os.path.isdir(os.path.join(c, "evcouplings"))), _CANDIDATES[-1])
_STUB_ROOTS = ("matplotlib", "seaborn", "bokeh", "billiard", "Bio", "mpl_toolkits")


def available():
    return os.path.isdir(os.path.join(REFERENCE_ROOT, "evcouplings"))


class _StubLoader(importlib.abc.Loader):
    def create_module(self, spec):
        m = mock.MagicMock(name=spec.name)
        m.__name__ = spec.name
        m.__path__ = []
        m.__spec__ = spec
        m.__loader__ = self
        return m

    def exec_module(self, module):
        pass


class _StubFinder(importlib.abc.MetaPathFinder):
    def find_spec(self, fullname, path=None, target=None):
        if fullname.split(".")[0] in _STUB_ROOTS:
            return importlib.machinery.ModuleSpec(fullname, _StubLoader(), is_package=True)
        return None


def _install_ruamel_shim():
    try:
        import ruamel.yaml  # noqa: F401
        return
    except ImportError:
        pass
    import yaml
    ruamel = types.ModuleType("ruamel")
    ruamel.__path__ = []
    ry = types.ModuleType("ruamel.yaml")
    ry.__path__ = []
    ry.safe_load = yaml.safe_load
    ry.load = yaml.load
    ry.dump = yaml.dump
    ry.Dumper = yaml.Dumper
    ry.RoundTripLoader = yaml.SafeLoader
    ry.RoundTripDumper = yaml.Dumper
    ry.parser = yaml.parser
    ry.scanner = yaml.scanner
    comments = types.ModuleType("ruamel.yaml.comments")

    class CommentedBase(object):
        pass

    comments.CommentedBase = CommentedBase
    ry.comments = comments
    ruamel.yaml = ry
    sys.modules["ruamel"] = ruamel
    sys.modules["ruamel.yaml"] = ry
    sys.modules["ruamel.yaml.comments"] = comments


_installed = False


def install():
    """Make ``import evcouplings`` resolve to the unmodified reference."""
    global _installed
    if _installed:
        return
    if not available():
        raise RuntimeError("the reference is present neither at $EVC_REFERENCE nor in baseline/_ref")
    warnings.filterwarnings("ignore", category=SyntaxWarning)
    _install_ruamel_shim()
    if not any(isinstance(f, _StubFinder) for f in sys.meta_path):
        sys.meta_path.append(_StubFinder())
    if REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, REFERENCE_ROOT)
    _installed = True
