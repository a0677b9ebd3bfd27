"""The CPU stand-in of the C ABI (fake_backend.FakeContext) against the real binding ``_native.Context``: every public
method and property of the stand-in exists on the binding, a method with the same parameter names, so the host tests
cannot drive the Model through calls the library does not have.  Reads only the Python class (no library, no GPU)."""
import inspect

import pytest

import fake_backend
from openwakeword_b200 import _native

PUBLIC = sorted(k for k, v in vars(fake_backend.FakeContext).items()
                if not k.startswith("_") and (inspect.isfunction(v) or isinstance(v, property)))


def _params(f):
    return [p for p in inspect.signature(f).parameters if p != "self"]


@pytest.mark.parametrize("name", PUBLIC)
def test_the_binding_has_it(name):
    fake, real = vars(fake_backend.FakeContext)[name], inspect.getattr_static(_native.Context, name, None)
    assert real is not None, f"_native.Context has no {name}"
    assert isinstance(fake, property) == isinstance(real, property), name
    if inspect.isfunction(fake):
        assert _params(fake) == _params(real), name


def test_the_constructor_takes_the_bindings_arguments():
    assert _params(fake_backend.FakeContext.__init__) == _params(_native.Context.__init__)
