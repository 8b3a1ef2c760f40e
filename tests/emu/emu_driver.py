"""The model drivers of nabladft_b200 (subclasses of `_lib.EngineDriver`) as the emulation tests drive them.  TEST INFRASTRUCTURE ONLY."""
import ctypes


def load(name: str, prefixes) -> ctypes.CDLL:
    """The emulation build of nabladft_b200/csrc/<name>.cu with the prototypes of the symbols starting with `prefixes` bound."""
    from build_emu import build

    from nabladft_b200 import _lib

    lib = _lib.bind(ctypes.CDLL(build(name=name)), prefixes)
    lib.nb200_emu_check_guards.restype = ctypes.c_int32
    return lib


def poisoned(cls, emulated: bool = True, checked=()):
    """`cls` with every buffer its `_buffer` hands out filled with `fill` bytes (0xFF: NaN floats, -1 indices) before the call that uses it:
    device memory comes back uninitialised, fresh CPU pages are zero, so a kernel reading what it never wrote shows up here and not only on
    the GPU.  `emulated`: the calls take host tensors and no stream (the emulation build).  The methods named in `checked` are bracketed by
    the guard-zone check of the emulation build (see `guarded`)."""

    class Driver(cls):
        fill = 255

        if emulated:
            def _stream(self):
                return None

            def _on_device(self, t):
                return True

        def _buffer(self, attr, nbytes, device):
            buf = super()._buffer(attr, nbytes, device)
            buf.fill_(self.fill)
            return buf

        def guarded(self, fn, *a, **kw):
            """fn(*a, **kw), after which no guard zone behind a workspace array may have been overwritten and some must have been registered."""
            self.lib.nb200_emu_check_guards()  # forget the zones of earlier calls: their buffers may be gone
            out = fn(*a, **kw)
            n = self.lib.nb200_emu_check_guards()
            assert n < 0, f"{n} guard zones behind workspace arrays were overwritten" if n > 0 else "no guard zones were registered"
            return out

    def checked_method(name):
        method = getattr(cls, name)
        return lambda self, *a, **kw: self.guarded(method.__get__(self), *a, **kw)

    for name in checked:
        setattr(Driver, name, checked_method(name))
    Driver.__name__ = Driver.__qualname__ = ("Emu" if emulated else "Poison") + cls.__name__
    return Driver
