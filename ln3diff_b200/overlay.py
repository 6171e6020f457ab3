"""Route the reference's own import names to this package -- the drop-in switch.

The reference scripts (`scripts/vit_triplane_diffusion_sample*.py`) run from the repository root with
`sys.path.append('.')` and import its packages by their top-level names (`dit.dit_trilatent`,
`sgm.modules.diffusionmodules.sampling`, `nsr.volumetric_rendering.renderer`, ...).  `install()` puts an
import hook in front of the normal path finders that answers exactly the module names this package
mirrors (MIRRORED below) with the `ln3diff_b200.*` implementation and leaves every other name --
parent packages, datasets, conditioners, training utilities -- to the reference checkout on `sys.path`:

    import ln3diff_b200.overlay as overlay
    overlay.install()                      # before the reference modules are imported
    from dit.dit_trilatent import DiT_models        # -> ln3diff_b200.dit.dit_trilatent
    from nsr.train_util_diffusion import ...        # -> the untouched reference file

The mirrors export the hot-path subset of each module.  Names they do not define -- the reference's other
classes of the same file (`ViTTriplaneDecomposed`, `Encoder`, `MVEncoder`, `ImageCondDiTBlock`, ...) that
`nsr/script_util.py` / `guided_diffusion/script_util.py` import next to the mirrored ones -- fall back to the
reference's own file: while the hook is installed every mirror module carries a module-level `__getattr__`
(PEP 562) that loads the reference module of the same name in a "reference world" (hook off, aliases out of
`sys.modules`, so the reference file sees its own sibling modules) and delegates to it.

`uninstall()` removes the hook, the fallbacks and the aliases it created.  Nothing is copied or patched on disk.
"""
from __future__ import annotations

import importlib
import importlib.abc
import importlib.util
import sys
import threading

# reference module name -> mirror (one line per file of the hot path)
MIRRORED = {
    "dit.dit_trilatent": "ln3diff_b200.dit.dit_trilatent",
    "dit.dit_i23d": "ln3diff_b200.dit.dit_i23d",
    "dit.dit_decoder": "ln3diff_b200.dit.dit_decoder",
    "dit.dit_models_xformers": "ln3diff_b200.dit.dit_models_xformers",
    "sgm.modules.diffusionmodules.sampling": "ln3diff_b200.sgm.modules.diffusionmodules.sampling",
    "sgm.modules.diffusionmodules.sampling_utils": "ln3diff_b200.sgm.modules.diffusionmodules.sampling_utils",
    "sgm.modules.diffusionmodules.denoiser": "ln3diff_b200.sgm.modules.diffusionmodules.denoiser",
    "sgm.modules.diffusionmodules.denoiser_scaling": "ln3diff_b200.sgm.modules.diffusionmodules.denoiser_scaling",
    "sgm.modules.diffusionmodules.discretizer": "ln3diff_b200.sgm.modules.diffusionmodules.discretizer",
    "sgm.modules.diffusionmodules.guiders": "ln3diff_b200.sgm.modules.diffusionmodules.guiders",
    "guided_diffusion.gaussian_diffusion": "ln3diff_b200.guided_diffusion.gaussian_diffusion",
    "guided_diffusion.respace": "ln3diff_b200.guided_diffusion.respace",
    "transport": "ln3diff_b200.transport",
    "transport.transport": "ln3diff_b200.transport.transport",
    "nsr.triplane": "ln3diff_b200.nsr.triplane",
    "nsr.volumetric_rendering.renderer": "ln3diff_b200.nsr.volumetric_rendering.renderer",
    "nsr.volumetric_rendering.ray_sampler": "ln3diff_b200.nsr.volumetric_rendering.ray_sampler",
    "vit.vit_triplane": "ln3diff_b200.vit.vit_triplane",
    "ldm.modules.diffusionmodules.model": "ln3diff_b200.ldm.modules.diffusionmodules.model",
}


_REFERENCE: dict = {}          # reference module name -> the reference's own module object (private, lazily loaded)
_lock = threading.RLock()


def reference_module(fullname: str):
    """The reference's own implementation of a mirrored module name, imported from the checkout on `sys.path`
    with the hook disabled and every alias out of `sys.modules` for the duration (so the file resolves its
    sibling imports -- `from .dit_models_xformers import *` -- against reference files, not mirrors).  The
    modules this pulls in under mirrored names are moved to a private table; the aliases are restored."""
    with _lock:
        mod = _REFERENCE.get(fullname)
        if mod is not None:
            return mod
        saved = {n: sys.modules.pop(n) for n in MIRRORED if n in sys.modules}
        was = _finder.enabled if _finder is not None else False
        if _finder is not None:
            _finder.enabled = False
        try:
            for n, m in _REFERENCE.items():          # reference modules already loaded stay visible to each other
                sys.modules[n] = m
            importlib.import_module(fullname)
            for n in MIRRORED:
                if n in sys.modules:
                    _REFERENCE[n] = sys.modules[n]
        finally:
            for n in MIRRORED:
                sys.modules.pop(n, None)
            sys.modules.update(saved)
            if _finder is not None:
                _finder.enabled = was
        return _REFERENCE[fullname]


def _make_fallback(refname: str):
    def __getattr__(name: str):
        if name.startswith("__") and name.endswith("__"):
            raise AttributeError(name)
        try:
            ref = reference_module(refname)
        except ImportError as e:
            raise AttributeError(f"{refname}.{name}: not mirrored by ln3diff_b200, and the reference module could not "
                                 f"be imported from sys.path ({e})") from e
        try:
            v = getattr(ref, name)
        except AttributeError:
            raise AttributeError(f"module '{refname}' (ln3diff_b200 mirror + reference fallback) has no attribute '{name}'")
        # a name the reference file merely re-exports from ANOTHER mirrored module (vit.vit_triplane's
        # `Triplane` is nsr.triplane's) must resolve to that module's mirror, not to the reference-world object
        home = MIRRORED.get(getattr(v, "__module__", None) or "")
        if home is not None:
            mirrored = importlib.import_module(home).__dict__.get(getattr(v, "__name__", name))
            if mirrored is not None:
                return mirrored
        return v
    return __getattr__


class _AliasLoader(importlib.abc.Loader):
    def __init__(self, target: str, refname: str):
        self.target, self.refname = target, refname

    def create_module(self, spec):
        m = importlib.import_module(self.target)         # the mirror module object itself
        if "__getattr__" not in m.__dict__:
            m.__dict__["__getattr__"] = _make_fallback(self.refname)
            _patched.append(m)
        return m

    def exec_module(self, module):                       # already executed under its own name
        pass


_patched: list = []


class _MirrorFinder(importlib.abc.MetaPathFinder):
    enabled = True

    def find_spec(self, fullname, path=None, target=None):
        tgt = MIRRORED.get(fullname)
        if tgt is None or not self.enabled:
            return None
        is_pkg = tgt == "ln3diff_b200.transport"
        spec = importlib.util.spec_from_loader(fullname, _AliasLoader(tgt, fullname), is_package=is_pkg)
        if is_pkg:
            spec.submodule_search_locations = list(importlib.import_module(tgt).__path__)
        return spec


_finder: _MirrorFinder | None = None


def install() -> None:
    """Install the import hook (idempotent).  Reference modules of MIRRORED that were imported before this
    call stay what they were: call it first."""
    global _finder
    if _finder is None:
        _finder = _MirrorFinder()
        sys.meta_path.insert(0, _finder)


def uninstall() -> None:
    global _finder
    if _finder is not None:
        sys.meta_path.remove(_finder)
        _finder = None
    for m in _patched:
        m.__dict__.pop("__getattr__", None)
    _patched.clear()
    _REFERENCE.clear()
    for name, tgt in MIRRORED.items():
        m = sys.modules.get(name)
        if m is not None and getattr(m, "__name__", None) == tgt:
            del sys.modules[name]
