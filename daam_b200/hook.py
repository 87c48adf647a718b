"""Context-managed monkey patching (the reference's L0, ``daam/hook.py:22-86``).

``ObjectHooker`` wraps one object: ``hook()`` runs the subclass' ``_hook_impl`` (which typically calls
``monkey_patch``), ``unhook()`` puts every replaced attribute back and runs ``_unhook_impl``; both are also reachable
as a ``with`` block. ``AggregateHooker`` does the same for a list of hookers. Public names, call signatures and the
two error messages (``'Already hooked module'``, ``'Module is not hooked'``, hook.py:36-37, 46-47) are the
reference's, because user code and the tracer rely on them; the layer walker lives in ``locate.py`` and is re-exported
here under its reference name.
"""
from __future__ import annotations

import functools
from typing import Any, Callable, Dict, Generic, List, TypeVar

from .locate import ModuleLocator, UNetCrossAttentionLocator

__all__ = ['ObjectHooker', 'ModuleLocator', 'AggregateHooker', 'UNetCrossAttentionLocator']

ModuleType = TypeVar('ModuleType')
ModuleListType = TypeVar('ModuleListType', bound=List)


class ObjectHooker(Generic[ModuleType]):
    def __init__(self, module: ModuleType):
        self.module: ModuleType = module
        self.hooked: bool = False
        self._replaced: Dict[str, Any] = {}     # attribute name -> what it was before monkey_patch

    # -- lifecycle ----------------------------------------------------------------------------------------------------
    def hook(self):
        if self.hooked:
            raise RuntimeError('Already hooked module')
        self.hooked = True
        self._replaced = {}
        self._hook_impl()
        return self

    def unhook(self):
        if not self.hooked:
            raise RuntimeError('Module is not hooked')
        while self._replaced:
            name, original = self._replaced.popitem()
            setattr(self.module, name, original)
        self.hooked = False
        self._unhook_impl()
        return self

    def __enter__(self):
        return self.hook()

    def __exit__(self, exc_type, exc_val, exc_tb):
        self.unhook()

    # -- patching helpers for subclasses -------------------------------------------------------------------------------
    def monkey_patch(self, fn_name: str, fn: Callable, strict: bool = True):
        """``module.fn_name`` becomes ``fn(module, *args, **kwargs)``. With ``strict=False`` an attribute the object
        does not have is skipped silently (SDXL pipelines have no safety checker)."""
        if not hasattr(self.module, fn_name):
            if strict:
                raise AttributeError(f'{type(self.module).__name__!r} object has no attribute {fn_name!r}')
            return
        self._replaced.setdefault(fn_name, getattr(self.module, fn_name))
        setattr(self.module, fn_name, functools.partial(fn, self.module))

    def monkey_super(self, fn_name: str, *args, **kwargs):
        """Call what ``fn_name`` was before it got patched."""
        return self._replaced[fn_name](*args, **kwargs)

    # -- to be provided by subclasses -------------------------------------------------------------------------------------
    def _hook_impl(self):
        raise NotImplementedError

    def _unhook_impl(self):
        pass


class AggregateHooker(ObjectHooker[ModuleListType]):
    """Hooks / unhooks every hooker of ``self.module`` (a list), in order."""

    def register_hook(self, hook: ObjectHooker):
        self.module.append(hook)

    def _hook_impl(self):
        for member in self.module:
            member.hook()

    def _unhook_impl(self):
        for member in self.module:
            member.unhook()
