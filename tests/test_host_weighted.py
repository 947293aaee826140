"""CPU tests (no GPU) of the per-pixel weighted projection: the weighted oracle, the binding's routing and checks, the
sharding of the weights, the per-layer checker on an emulation of the weighted last-layer forward (and its seeded
defects), and the plans of the fp16 path's weighted last-layer forward (host code of the CUDA library)."""
import ctypes
import os
import socket

import numpy as np
import pytest
import torch

import layer_ref as R
import weighted_layer_ref as WR
import weighted_oracle as WO
from oracle import defensegan_oracle as O
from test_host_layers import Emu, N_PAD, N_ROWS
from test_host_widths import GRID, _desc

from recording import cpu_native  # noqa: F401  (the fixture)


# ---- the weighted oracle ----

def _problem(arch="mnist", b=2, rr=2, latent=16, net_dim=8, seed=3):
    w = O.init_generator_weights(arch, latent_dim=latent, net_dim=net_dim, random_bias=True)
    x = O.synthetic_images(arch, w, b, kind="S2", seed=seed, latent_dim=latent)
    z = O.sample_z0(b * rr, latent, seed=seed)
    return w, x, z


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_oracle_unit_weights_are_the_unweighted_bits(arch):
    w, x, z = _problem(arch)
    ones = np.ones_like(x)
    for a, b in zip(WO.loss_and_grad(arch, w, x, z, 2, pixel_weights=ones), O.loss_and_grad(arch, w, x, z, 2)):
        assert np.array_equal(a, b)
    got = WO.reconstruct(arch, w, x, 2, 3, z_init_val=z, pixel_weights=ones)
    want = O.reconstruct(arch, w, x, 2, 3, z_init_val=z)
    for k in ("rec", "loss_min", "idx", "loss_all", "rec_all", "z_final"):
        assert np.array_equal(got[k], want[k]), k


def test_oracle_weighted_gradient_matches_central_differences():
    w, x, z = _problem(b=1, rr=2, latent=8)
    pw = np.random.RandomState(1).uniform(0, 1, size=x.shape)
    pw[..., :5, :] = 0
    _, _, g = WO.loss_and_grad("mnist", w, x, z, 2, dtype=torch.float64, pixel_weights=pw)
    h = 1e-6
    num = np.zeros_like(g)
    for r in range(z.shape[0]):
        for k in range(z.shape[1]):
            zp, zm = z.astype(np.float64).copy(), z.astype(np.float64).copy()
            zp[r, k] += h
            zm[r, k] -= h
            lp = WO.loss_and_grad("mnist", w, x, zp, 2, dtype=torch.float64, pixel_weights=pw)[1].sum()
            lm = WO.loss_and_grad("mnist", w, x, zm, 2, dtype=torch.float64, pixel_weights=pw)[1].sum()
            num[r, k] = (lp - lm) / (2 * h)
    np.testing.assert_allclose(g, num, rtol=1e-6, atol=1e-10)


def test_oracle_ignores_pixels_of_weight_zero():
    w, x, z = _problem(b=2, rr=2)
    pw = (np.random.RandomState(2).uniform(0, 1, size=x.shape) > 0.5).astype(np.float32)
    x2 = np.where(pw == 0, np.random.RandomState(4).uniform(0, 1, size=x.shape), x).astype(np.float32)
    assert not np.array_equal(x, x2)
    for a, b in zip(WO.loss_and_grad("mnist", w, x, z, 2, pixel_weights=pw), WO.loss_and_grad("mnist", w, x2, z, 2, pixel_weights=pw)):
        assert np.array_equal(a, b)
    a = WO.reconstruct("mnist", w, x, 2, 3, z_init_val=z, pixel_weights=pw)
    b = WO.reconstruct("mnist", w, x2, 2, 3, z_init_val=z, pixel_weights=pw)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_oracle_all_zero_weights_keep_z0_and_choose_restart_0():
    w, x, z = _problem(b=2, rr=3)
    got = WO.reconstruct("mnist", w, x, 3, 3, z_init_val=z, pixel_weights=np.zeros_like(x))
    assert np.array_equal(got["z_final"], z) and list(got["idx"]) == [0, 0] and not got["loss_all"].any()


# ---- the C-ABI and the binding ----

class FakeOut:
    """The `out` buffer of reconstruct as the binding checks it (a contiguous CUDA float32 tensor shaped like x)."""
    is_cuda, dtype = True, torch.float32

    def __init__(self, n):
        self.n = n

    def is_contiguous(self):
        return True

    def numel(self):
        return self.n

    def data_ptr(self):
        return 0


def test_binding_routes_only_weighted_calls_to_the_weighted_entries(cpu_native):
    x = torch.rand(2, 28, 28, 1)
    cpu_native.reconstruct(x, 3, 5, out=FakeOut(x.numel()))
    cpu_native.loss_grad(x, torch.zeros(6, 8), 3)
    assert [c[0] for c in cpu_native.lib.calls] == ["dgan_workspace_bytes", "dgan_reconstruct",
                                                    "dgan_workspace_bytes", "dgan_loss_grad"]
    cpu_native.lib.calls.clear()
    w = torch.rand(2, 28, 28, 1)
    cpu_native.reconstruct(x, 3, 5, pixel_weights=w, out=FakeOut(x.numel()))
    cpu_native.loss_grad(x, torch.zeros(6, 8), 3, pixel_weights=w)
    calls = cpu_native.lib.calls
    assert [c[0] for c in calls] == ["dgan_workspace_bytes_weighted", "dgan_reconstruct_weighted",
                                     "dgan_workspace_bytes_weighted", "dgan_loss_grad_weighted"]
    assert calls[1][1][3].value == w.data_ptr() and calls[3][1][2].value == w.data_ptr()
    with pytest.raises(ValueError, match="pixel_weights"):
        cpu_native.reconstruct(x, 3, 5, pixel_weights=torch.rand(1, 28, 28, 1))
    assert len(calls) == 4


class FakeNative:
    def __init__(self):
        self.calls = []

    def reconstruct(self, x, *args, **kw):
        self.calls.append((x, args, kw))
        return x


def _gan():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    fake = FakeNative()
    gan._as_cuda = lambda t: torch.as_tensor(t).to(torch.float32)
    gan._get_native = lambda device: fake
    return gan, fake


def test_defensegan_reconstruct_without_weights_calls_as_before():
    gan, fake = _gan()
    x = torch.rand(2, 28, 28, 1)
    gan.reconstruct(x)
    (_, args, kw), = fake.calls
    assert sorted(kw) == ["decay_lr", "momentum", "out", "return_aux", "seed", "z_init_val", "z_row_offset"]


def test_defensegan_reconstruct_broadcasts_the_weights_once():
    gan, fake = _gan()
    x = torch.rand(2, 28, 28, 1)
    mask = np.zeros((28, 28, 1), dtype=np.float32)
    mask[:14] = 1
    gan.reconstruct(x, pixel_weights=mask)
    pw = fake.calls[0][2]["pixel_weights"]
    assert pw.shape == x.shape and pw.is_contiguous() and torch.equal(pw[1], torch.as_tensor(mask))


@pytest.mark.parametrize("bad,match", [(np.ones((3, 28, 28, 1)), "broadcast"), (np.full((28, 28, 1), np.nan), "finite"),
                                       (np.full((28, 28, 1), 1.5), r"\[0, 1\]"), (np.full((28, 28, 1), -0.1), r"\[0, 1\]"),
                                       (np.full((28, 28, 1), np.inf), "finite")])
def test_bad_weights_raise_before_any_native_call(bad, match):
    gan, fake = _gan()
    counter = gan._call_counter
    with pytest.raises(ValueError, match=match):
        gan.reconstruct(torch.rand(2, 28, 28, 1), pixel_weights=bad)
    assert fake.calls == [] and gan._call_counter == counter


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _gloo_worker(rank, world, port, n_images, rec_rr, ret):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from defensegan_b200.parallel import sharded_apply
        g = torch.Generator().manual_seed(0)
        images = torch.rand(n_images, 2, 2, 1, generator=g)
        weights = torch.rand(n_images, 2, 2, 1, generator=g)

        def local_fn(x, z, out, first_image, pixel_weights):
            # stand-in for the per-rank weighted projection: depends on the image and its weights
            out.copy_(x * pixel_weights + first_image * 0)

        got = sharded_apply(local_fn, images, rec_rr, pixel_weights=weights)
        ok = bool(torch.equal(got, images * weights))
        # a weight map that broadcasts (one for all images) is sliced after broadcasting
        got = sharded_apply(local_fn, images, rec_rr, pixel_weights=weights[:1])
        ret[rank] = ok and bool(torch.equal(got, images * weights[:1]))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n_images", [8, 5])
def test_sharding_slices_the_weights_with_the_images_gloo_world2(n_images):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, n_images, 3, ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert ret[0] and ret[1]


# ---- the per-layer checker on the weighted last-layer forward ----

class WeightedEmu(Emu):
    """Emu with the weighted last-layer forward (e = w (y - x): loss part e (y - x), d(pre) RN16(gscale e act'(y))) and the
    backward from its d(pre).  Defects: the weight ignored, applied twice, the next row's weights, or applied to the loss
    but not to d(pre)."""

    def __init__(self, defect=None):
        super().__init__(defect)
        g = torch.Generator().manual_seed(9)
        self.wpix = torch.rand(N_ROWS, 784, generator=g)
        self.wpix[:, ::7] = 0

    def run(self):
        ws = super().run()
        y = ws["y"]                                                  # [n_pad][784]
        rows = lambda t: torch.cat([t, t[-1:].expand(N_PAD - N_ROWS, -1)])
        x, w = rows(self.x), rows(self.wpix)
        if self._d("last.fwd", "ignored"):
            w = torch.ones_like(w)
        elif self._d("last.fwd", "neighbour"):
            w = torch.roll(w, -1, dims=0)
        d = y - x
        e = w * d
        if self._d("last.fwd", "twice"):
            e = w * e
        de = d if self._d("last.fwd", "loss_only") else e
        dpre = (de * (y * (1 - y)) * R.GRAD_SCALE).half()
        blk, k = R.block_perm(28, 1, torch.device("cpu"))
        dblk = torch.zeros(49, N_PAD, 16, dtype=torch.float16)
        dblk[blk, :, k] = dpre.t()
        lp = torch.zeros(49, N_PAD)
        lp.index_add_(0, blk, (e * d).t())
        ws["dblk"], ws["loss_part"] = dblk, lp
        self.backward(ws)
        return ws

    def check(self, ws):
        stats = R.Stats()
        R.check_inputs(self.net, ws, N_ROWS, self.z)
        R.check_forward(self.net, ws, N_ROWS, stats, "")
        WR.check_last_fwd_weighted(self.net, ws, N_ROWS, self.x, self.wpix, stats, "")
        R.check_backward(self.net, ws, N_ROWS, stats, "")
        return stats


def test_checker_accepts_a_weighted_emulation():
    stats = WeightedEmu().check(WeightedEmu().run())
    assert any(k.startswith("last.fwd (dblk)") for k in stats.rows)


@pytest.mark.parametrize("kind", ["ignored", "twice", "neighbour", "loss_only"])
def test_checker_rejects_a_seeded_weighting_defect(kind):
    emu = WeightedEmu(defect=("last.fwd", kind))
    with pytest.raises(AssertionError, match=r"last\.fwd"):
        emu.check(emu.run())


# ---- plans of the weighted last-layer forward (dgan_debug_check_weighted_plans) ----

def _check_weighted(arch, latent, net_dim, use_bn, n_rows, n_pairs=66, mutate=0):
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_check_weighted_plans.restype = ctypes.c_int
    lib.dgan_debug_check_weighted_plans.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dgan_last_error.restype = ctypes.c_char_p
    d = _desc(arch, latent, net_dim, use_bn)
    rc = lib.dgan_debug_check_weighted_plans(ctypes.byref(d), n_rows, n_pairs, mutate)
    return rc, (lib.dgan_last_error() or b"").decode()


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", GRID + [("mnist", 128, 64, 0), ("celeba", 128, 64, 0),
                                                               ("mnist", 128, 64, 1)])
@pytest.mark.parametrize("n_rows", [1, 300, 2560])
def test_weighted_plans_pass_the_validator(arch, latent, net_dim, use_bn, n_rows):
    rc, msg = _check_weighted(arch, latent, net_dim, use_bn, n_rows)
    assert rc == 0, msg


@pytest.mark.parametrize("arch,latent,net_dim,use_bn", [("mnist", 128, 64, 0), ("celeba", 200, 48, 0), ("mnist", 128, 64, 1)])
def test_validator_names_the_damaged_weighted_direction(arch, latent, net_dim, use_bn):
    for mutate in range(1, 12):
        rc, msg = _check_weighted(arch, latent, net_dim, use_bn, 2560, mutate=mutate)
        assert rc != 0 and msg.startswith("last.fwd.w:"), (mutate, rc, msg)
