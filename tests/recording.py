"""The CPU tests' recording stand-ins for the CUDA library: a NativeGenerator whose library records every call, a CUDA
`out` tensor, and a DefenseGAN model whose native generator records the keyword arguments it is called with.  Import
`cpu_native` into a test module to use it as a fixture."""
import contextlib
import ctypes

import pytest
import torch


class FakeLib:
    """Stands in for the CUDA library under NativeGenerator: records every entry point it is called through."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append((name, args))
            return 1 << 20 if name.startswith("dgan_workspace_bytes") else 0
        return fn


class Out:
    """Stands in for a CUDA `out` tensor of n elements."""
    is_cuda, dtype = True, torch.float32

    def __init__(self, n):
        self.n = n

    def is_contiguous(self):
        return True

    def numel(self):
        return self.n

    def data_ptr(self):
        return 0


@pytest.fixture
def cpu_native(monkeypatch):
    """A NativeGenerator (MNIST, latent 8) on the CPU whose library is a FakeLib.  `calls` holds the library calls, and
    `seen` the tensors it converted for the library, by argument name."""
    from defensegan_b200 import _native
    seen = {}

    def converter(dtype):
        def convert(t, name):
            seen[name] = t.to(dtype).contiguous()
            return seen[name]
        return convert

    class Stream:
        cuda_stream = 0

    monkeypatch.setattr(_native, "_require_cuda_f32", converter(torch.float32))
    monkeypatch.setattr(_native, "_require_cuda_i32", converter(torch.int32))
    monkeypatch.setattr(_native, "_require_aligned_out", lambda rec: None)
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "current_stream", lambda d=None: Stream())
    g = object.__new__(_native.NativeGenerator)
    g.lib, g.device, g._ws, g._handle = FakeLib(), torch.device("cpu"), None, ctypes.c_void_p(0)
    g.image_dim, g.hwc, g.latent_dim, g.use_bn = (28, 28, 1), 784, 8, False
    g.calls, g.seen, g.Out = g.lib.calls, seen, Out
    return g


def recording_gan(**kw):
    """(MNIST model with rec_rr 4 and rec_iters 50, [(method, kwargs)] of each reconstruct / reconstruct_measured call
    its native generator receives)."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, **kw)
    seen = []

    class FakeNative:
        def reconstruct(self, x, *args, **kw):
            seen.append(("reconstruct", kw))
            return x

        def reconstruct_measured(self, y, a, *args, **kw):
            seen.append(("reconstruct_measured", kw))
            return y

    gan._as_cuda = lambda t: t.to(torch.float32)
    gan._get_native = lambda device: FakeNative()
    gan.rec_rr, gan.rec_iters = 4, 50
    return gan, seen
