"""GPU tests (H100, -m gpu) of the Adam update of the latent rows (dgan_reconstruct_adam, dgan_reconstruct_measured_adam,
dgan_reconstruct_measured_csr_adam), on MNIST and CelebA, fp32 and fp16, with BatchNorm where it applies:
  - the update on its stored operands: after L = 2 the workspace's g, m (in v), s, z and z_h against fp64 from the stored
    partial sums, then L = 3 from the same z0 against the first call's m, s and z (the bias correction at k = 2); padded
    channels exactly 0 (and tile-padding rows, but on the fp16 image loss), z_h = RN16(z); image and measured loss;
  - R = 10, L = 200 against the fp64 Adam oracle (tests/adam_oracle.py) on the image loss and on the measured loss with
    dense and CSR operators;
  - bit identities: an identity prune schedule gives the unpruned bits, any schedule the result composed from rec_rr = 1
    calls, w = 1 the unweighted bits, fp32 CSR the dense bits; an image whose weights are all 0 keeps z0;
  - momentum and Adam calls alternating on one workspace give fresh handles' bits;
  - the header's launch and enqueue counts, and no allocation in steady state;
  - the layout: the momentum layout plus s."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import adam_oracle as AO
import layer_ref as LR
import measured_oracle as MO
from gpu_support import gsum as _gsum, option_layout as _layout, read as _read
from gpu_support import rec, rec_m, release_cached_memory  # noqa: F401
from gpu_support import bits as _bits, gen as _gen, images as _images, same as _same, z0 as _z0
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

HWC = {"mnist": 784, "celeba": 12288}
SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}
ADAM = (0.9, 0.999, 1e-8)
CASES = [(p, a) for p in ("fp32", "fp16") for a in ("mnist", "celeba")]
_rec, _rec_m = functools.partial(rec, adam=ADAM), functools.partial(rec_m, adam=ADAM)


# ---- the workspace ----

@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_adam_layout_is_the_momentum_layout_plus_s(precision):
    w, gen = _gen("celeba", precision, latent=100)
    try:
        B, R = 3, 4
        sched = [(5, 2), (9, 1)]
        for kw in (dict(), dict(weighted=1), dict(m=500), dict(m=500, nnz=7000)):
            _, mom = _layout(gen, B, R, adam=False, **kw)
            bufs, ada = _layout(gen, B, R, **kw)
            lines = ada.splitlines()
            assert "\n".join(lines[:-1]) + "\n" == mom, kw
            name, typ, off, *dims = lines[-1].split()
            n_pad = bufs["bufs"]["z"][2][0]
            assert (name, typ, dims) == ("s", "f32", [str(n_pad), "128"]), kw
            end = max(o + (int(np.prod(d)) * 4 + 1023) // 1024 * 1024 for t, o, d in _layout(gen, B, R, adam=False,
                                                                                              **kw)[0]["bufs"].values())
            assert int(off) == end, kw
        for weighted in (0, 1):
            _, mom = _layout(gen, B, R, weighted=weighted, sched=sched, adam=False)
            _, ada = _layout(gen, B, R, weighted=weighted, sched=sched)
            strip = lambda t: [ln for ln in t.splitlines() if not ln.startswith(("s ", "region "))]
            assert strip(ada) == strip(mom)
            assert sum(ln.startswith("s f32 ") for ln in ada.splitlines()) == len(sched) + 1
    finally:
        gen.close()


# ---- the update on its stored operands ----

def _check_update(ws1, ws2, z0p, lr, n, lat, tc, row_mul, pad_rows_zero, tag):
    """ws1 after L = 2 (step k = 1 from m = s = 0), ws2 after L = 3 (step k = 2 from ws1's m, s, z), each step against
    fp64 on the operands the kernel read: m and s from the stored partial sums and the previous step's stored m and s, to
    a few fp32 ulps of the sum of their terms' magnitudes (the terms of m may cancel); z from the previous z and this
    step's stored m and s, to a few ulps of z and of the step.  Padded latent channels exactly 0 (and, pad_rows_zero, the
    tile-padding rows); z_h = RN16(z)."""
    b1, b2, eps = (float(np.float32(v)) for v in ADAM)
    prev = dict(v=torch.zeros_like(ws1["v"]).double(), s=torch.zeros_like(ws1["s"]).double(), z=z0p.double())
    for k, ws in ((1, ws1), (2, ws2)):
        gg = (_gsum(ws["g"]) * row_mul).double()              # fp32 sum of the parts in order, times the multiplier
        c1, c2 = AO.adam_constants(lr, k - 1, b1, b2)
        m_ref = b1 * prev["v"] + (1 - b1) * gg
        m_abs = b1 * prev["v"].abs() + (1 - b1) * gg.abs()
        s_ref = b2 * prev["s"] + (1 - b2) * gg * gg
        m, s = ws["v"].double(), ws["s"].double()
        u_ref = c1 * m / (torch.sqrt(s) * c2 + eps)
        z_ref = prev["z"] - u_ref
        for name, got, ref, bound in (("m", ws["v"], m_ref, 4 * LR.half_ulp(m_abs, "f32")),
                                      ("s", ws["s"], s_ref, 4 * LR.half_ulp(s_ref, "f32")),
                                      ("z", ws["z"], z_ref, 2 * LR.half_ulp(prev["z"], "f32") +
                                       12 * LR.half_ulp(u_ref, "f32"))):
            err = (got.double() - ref).abs()
            bound = bound + 2.0 ** -149
            assert bool((err <= bound).all()), "%s k=%d %s: max err / bound %.3g" % (tag, k, name,
                                                                                     float((err / bound).max()))
            if pad_rows_zero:
                LR.check_pad_rows_zero("%s k=%d %s" % (tag, k, name), got, n)
            LR.check_zero_pad("%s k=%d %s" % (tag, k, name), got, lat)
        if tc:
            assert torch.equal(ws["z_h"], ws["z"].half()), "%s k=%d: z_h is not RN16(z)" % (tag, k)
        prev = dict(v=m, s=s, z=ws["z"].double())


@pytest.mark.parametrize("use_bn", [False, True])
@pytest.mark.parametrize("precision,arch", CASES)
def test_update_on_its_stored_operands(precision, arch, use_bn):
    lat, B, R, lr = 100, 3, 2, 0.01
    w, gen = _gen(arch, precision, use_bn=use_bn, latent=lat)
    tc = precision == "fp16"
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R, lat)
        names = ("g", "v", "s", "z") + (("z_h",) if tc else ())
        gmul = torch.tensor(2.0, dtype=torch.float32) / torch.tensor(float(HWC[arch]), dtype=torch.float32)
        if tc:
            gmul = gmul / torch.tensor(LR.GRAD_SCALE, dtype=torch.float32)
        bufs, _ = _layout(gen, B, R)
        out = []
        for L in (2, 3):
            _rec(gen, x, R, L, lr, z0)
            out.append({nm: _read(gen, bufs, nm) for nm in names})
        z0p = torch.zeros_like(out[0]["z"])
        z0p[:B * R, :lat] = z0
        # the fp16 image loss's last-layer forward leaves a gradient in the tile-padding rows, as on the momentum path,
        # so they move; they are never observed
        _check_update(out[0], out[1], z0p, lr, B * R, lat, tc, gmul.item(), not tc, "%s %s image" % (precision, arch))
        if use_bn:
            return
        # the measured loop: g with the cotangent's row scales divided out (fp16), unscaled (fp32)
        a = torch.tensor(MO.gaussian_operator(64, HWC[arch], seed=1)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        bufs, _ = _layout(gen, B, R, m=64)
        out = []
        for L in (2, 3):
            _rec_m(gen, y, a, R, L, lr, z0)
            out.append({nm: _read(gen, bufs, nm) for nm in names + ("mscale",)})
        for o in out:
            n_pad = o["z"].shape[0]
            scale = torch.ones(n_pad, 1, device="cuda")
            if tc:
                scale[:B * R, 0] = 1.0 / o["mscale"][:B * R]
            o["g"] = o["g"] * scale.unsqueeze(0)                 # exact: power-of-two scales
        _check_update(out[0], out[1], z0p, lr, B * R, lat, tc, 1.0, True, "%s %s measured" % (precision, arch))
    finally:
        gen.close()


# ---- against the fp64 oracle ----

# precision: (bound on max |loss_min - oracle| / max oracle loss_min, least share of images choosing the oracle's restart,
# bound on |rec - oracle| where they do).  On an H100 80GB HBM3 (700 W) with these seeds the worst cases were
# 6.0e-4, 1.0 and 6.5e-3 on fp32 (margins 3.3x, -, 3x) and 4.7e-3 and 6.5e-2 on fp16 (margins 6x and 2.3x), where 2 to 4
# images make the restart share too coarse to bound: the fp16 operands of 200 Adam steps pick among near-equal restarts.
PARITY_TOL = {"fp32": (2e-3, 0.75, 2e-2), "fp16": (3e-2, 0.0, 1.5e-1)}
LR_IMAGE = 0.005


@pytest.mark.parametrize("precision,arch", CASES)
def test_long_horizon_parity_with_the_fp64_oracle(precision, arch):
    B, R, L = (4, 10, 200) if arch == "mnist" else (2, 10, 200)
    w, gen = _gen(arch, precision)
    try:
        imgs = O.synthetic_images(arch, w, B)
        z0 = O.sample_z0(B * R, 128)
        ref = AO.reconstruct(arch, w, R, L, LR_IMAGE, ADAM, images=imgs, z_init_val=z0, device="cuda")
        rec, loss, idx = _rec(gen, torch.tensor(imgs).cuda(), R, L, LR_IMAGE, torch.tensor(z0).cuda())
        _compare(precision, "%s image" % arch, rec, loss, idx, ref)
        a = MO.block_average_operator(*SHAPE[arch], 2)
        y = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
        ref = AO.reconstruct(arch, w, R, L, LR_IMAGE, ADAM, operator=a, measurements=y, z_init_val=z0, device="cuda")
        at = torch.tensor(a).cuda()
        for op, name in ((at, "dense"), (at.to_sparse_csr(), "csr")):
            rec, loss, idx = _rec_m(gen, torch.tensor(y).cuda(), op, R, L, LR_IMAGE, torch.tensor(z0).cuda())
            _compare(precision, "%s measured %s" % (arch, name), rec, loss, idx, ref)
    finally:
        gen.close()


def _compare(precision, tag, rec, loss, idx, ref):
    rel_tol, agree_min, rec_tol = PARITY_TOL[precision]
    dl = np.abs(loss.cpu().numpy().astype(np.float64) - ref["loss_min"])
    rel = float(dl.max()) / max(float(np.abs(ref["loss_min"]).max()), 1e-3)
    agree = float((idx.cpu().numpy() == ref["idx"]).mean())
    print("%s %s: max|dloss| / max loss = %.3g (tol %.1g), restart agreement %.2f, max |rec - oracle| %.3g"
          % (precision, tag, rel, rel_tol, agree, float(np.abs(rec.cpu().numpy().reshape(ref["rec"].shape) - ref["rec"]).max())))
    assert rel <= rel_tol, tag
    assert agree >= agree_min, tag
    # where the restarts agree, the reconstructions agree to the loss's precision
    same = idx.cpu().numpy() == ref["idx"]
    if same.any():
        d = np.abs(rec.cpu().numpy().reshape(ref["rec"].shape)[same] - ref["rec"][same]).max()
        assert d <= rec_tol, (tag, d)


# ---- bit identities ----

def _composed(gen, x, R, L, lr, z0, prune, measured=None):
    """The pruned Adam call's result from rec_rr = 1 Adam calls on the tiled images (or measurements)."""
    B = x.shape[0]
    xt = x.repeat_interleave(R, dim=0)

    def call(n_it):
        if measured is not None:
            return _rec_m(gen, xt, measured, 1, n_it, lr, z0)
        return _rec(gen, xt, 1, n_it, lr, z0)
    loss_at = {it: call(it)[1].cpu().numpy() for it, _ in prune}
    rec_all, loss_all, _ = call(L)
    loss_all = loss_all.cpu().numpy()
    rec = torch.empty((B,) + tuple(rec_all.shape[1:]), device="cuda")
    loss, idx = torch.empty(B, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda")
    for i in range(B):
        alive = list(range(R))
        for it, keep in prune:
            ranked = sorted(alive, key=lambda r: (np.isnan(loss_at[it][i * R + r]), loss_at[it][i * R + r], r))
            alive = sorted(ranked[:keep])
        best = alive[0]
        for r in alive[1:]:
            if loss_all[i * R + r] < loss_all[i * R + best]:
                best = r
        rec[i], loss[i], idx[i] = rec_all[i * R + best], float(loss_all[i * R + best]), best
    return [rec, loss, idx]


@pytest.mark.parametrize("precision,arch", CASES)
def test_bit_identities(precision, arch):
    B, R, L, lr = 4, 4, 12, 0.02
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        plain = _rec(gen, x, R, L, lr, z0)
        assert bool(torch.isfinite(plain[1]).all())
        # an identity schedule gives the unpruned bits; any schedule the composed result
        for sched in ([(5, R)], [(1, R), (6, R), (11, R)]):
            assert _same(_rec(gen, x, R, L, lr, z0, prune=sched), plain), sched
        for sched in ([(5, 2)], [(3, 3), (6, 2), (9, 1)]):
            assert _same(_rec(gen, x, R, L, lr, z0, prune=sched), _composed(gen, x, R, L, lr, z0, sched)), sched
        # w = 1 gives the unweighted bits, pruned or not
        ones = torch.ones_like(x)
        assert _same(_rec(gen, x, R, L, lr, z0, pixel_weights=ones), plain)
        assert _same(_rec(gen, x, R, L, lr, z0, pixel_weights=ones, prune=[(5, 2)]), _rec(gen, x, R, L, lr, z0,
                                                                                        prune=[(5, 2)]))
        # an image whose weights are all 0 keeps z0: its result is that of L = 1 (no update), restart 0, loss 0
        pw = torch.rand(x.shape, generator=torch.Generator().manual_seed(4)).cuda()
        pw[1] = 0
        got = _rec(gen, x, R, L, lr, z0, pixel_weights=pw)
        first = _rec(gen, x, R, 1, lr, z0, pixel_weights=pw)
        assert torch.equal(_bits(got[0][1]), _bits(first[0][1]))
        assert float(got[1][1]) == 0.0 and int(got[2][1]) == 0
        # the measured loss: identity schedule, composed result, and fp32 CSR = dense
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        mplain = _rec_m(gen, y, a, R, L, lr, z0)
        assert bool(torch.isfinite(mplain[1]).all())
        assert _same(_rec_m(gen, y, a, R, L, lr, z0, prune=[(1, R), (6, R)]), mplain)
        assert _same(_rec_m(gen, y, a, R, L, lr, z0, prune=[(5, 2)]), _composed(gen, y, R, L, lr, z0, [(5, 2)], a))
        acsr = a.to_sparse_csr()
        if precision == "fp32":
            assert _same(_rec_m(gen, y, acsr, R, L, lr, z0), mplain)
            assert _same(_rec_m(gen, y, acsr, R, L, lr, z0, prune=[(5, 2)]), _rec_m(gen, y, a, R, L, lr, z0, prune=[(5, 2)]))
        else:
            assert _same(_rec_m(gen, y, acsr, R, L, lr, z0, prune=[(1, R)]), _rec_m(gen, y, acsr, R, L, lr, z0))
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_bn_adam_runs_and_pruning_with_bn_is_refused(precision):
    from defensegan_b200 import _native
    B, R, L = 3, 2, 6
    w, gen = _gen("mnist", precision, use_bn=True)
    try:
        x = _images("mnist", w, B)
        z0 = _z0(B * R)
        got = _rec(gen, x, R, L, 0.01, z0)
        assert bool(torch.isfinite(got[1]).all())
        assert _same(_rec(gen, x, R, L, 0.01, z0), got)
        sched = (_native.dgan_prune_point * 1)(_native.dgan_prune_point(2, 1))
        assert gen.lib.dgan_workspace_bytes_adam(gen._handle, B, R, 0, sched, 1) == 0
        ws, need = gen._workspace(B, R, adam=True)
        prm = _native.dgan_rec_params(B, R, L, 0.01, 0.7, 0, 0, 0)
        ap = _native.dgan_adam_params(*ADAM)
        out = torch.empty_like(x)
        rc = gen.lib.dgan_reconstruct_adam(gen._handle, ctypes.byref(prm), ctypes.byref(ap), sched, 1, _native._ptr(x), None,
                                           _native._ptr(z0), _native._ptr(out), None, None, ws, need,
                                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == -3
    finally:
        gen.close()


# ---- calls on one handle, counts, steady state ----

@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_graph_cache_counts_and_steady_state(precision):
    arch, B, R, L = "mnist", 5, 3, 7
    w, gen = _gen(arch, precision)
    _, fresh_m = _gen(arch, precision)
    _, fresh_a = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.gaussian_operator(100, 784, seed=1)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()

        def call(g, kind):
            if kind == "mom":
                return _rec(g, x, R, L, 0.5, z0, adam=None)
            if kind == "adam":
                return _rec(g, x, R, L, 0.02, z0)
            if kind == "adam2":
                return _rec(g, x, R, L, 0.02, z0, adam=(0.5, 0.9, 1e-6))
            if kind == "madam":
                return _rec_m(g, y, a, R, L, 0.02, z0)
            return _rec_m(g, y, a, R, L, 0.5, z0, adam=None)

        want = {k: call(fresh_m if k in ("mom", "mmom") else fresh_a, k) for k in ("mom", "adam", "adam2", "madam", "mmom")}
        assert not _same(want["adam"], want["adam2"])
        for kind in ("adam", "mom", "adam", "adam2", "mom", "madam", "mmom", "madam", "adam"):
            assert _same(call(gen, kind), want[kind]), kind
        extra = (L - 1) if precision == "fp16" else 0
        for mk, ak in (("mom", "adam"), ("mmom", "madam")):
            call(gen, mk)
            enq, launches = gen.last_enqueue_count, gen.last_launch_count
            call(gen, ak)
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            for _ in range(3):
                call(gen, ak)
                assert gen.last_enqueue_count == enq, ak
                assert gen.last_launch_count == launches + (extra if ak == "adam" else 0), ak
            torch.cuda.synchronize()
            assert torch.cuda.mem_get_info()[0] == free0
        # pruned: the momentum counterpart's counts (+ L - 1 on the fp16 image loss)
        for kw in (dict(prune=[(3, 2)]), dict(prune=[(2, 2), (5, 1)], pixel_weights=torch.ones_like(x))):
            _rec(gen, x, R, L, 0.5, z0, adam=None, **kw)
            enq, launches = gen.last_enqueue_count, gen.last_launch_count
            _rec(gen, x, R, L, 0.02, z0, **kw)
            assert gen.last_enqueue_count == enq and gen.last_launch_count == launches + extra
        _rec_m(gen, y, a, R, L, 0.5, z0, adam=None, prune=[(3, 2)])
        enq, launches = gen.last_enqueue_count, gen.last_launch_count
        _rec_m(gen, y, a, R, L, 0.02, z0, prune=[(3, 2)])
        assert gen.last_enqueue_count == enq and gen.last_launch_count == launches
    finally:
        for g in (gen, fresh_m, fresh_a):
            g.close()


def test_bad_adam_parameters_are_refused_before_anything_is_enqueued():
    from defensegan_b200 import _native
    B, R, L = 2, 2, 4
    w, gen = _gen("mnist", "fp32")
    try:
        x = _images("mnist", w, B)
        z0 = _z0(B * R)
        ws, need = gen._workspace(B, R, adam=True)
        prm = _native.dgan_rec_params(B, R, L, 0.01, 0.7, 0, 0, 0)
        out = torch.full_like(x, 7.0)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        for bad in ((1.0, 0.999, 1e-8), (-0.1, 0.999, 1e-8), (0.9, 1.0, 1e-8), (0.9, float("nan"), 1e-8), (0.9, 0.999, 0.0),
                    (0.9, 0.999, float("inf")), (0.9, 0.999, -1e-8)):
            ap = _native.dgan_adam_params(*bad)
            rc = gen.lib.dgan_reconstruct_adam(gen._handle, ctypes.byref(prm), ctypes.byref(ap), None, 0, _native._ptr(x),
                                               None, _native._ptr(z0), _native._ptr(out), None, None, ws, need, stream)
            assert rc == -1, bad
            assert b"Adam" in gen.lib.dgan_last_error()
        torch.cuda.synchronize()
        assert bool((out == 7.0).all())
        with pytest.raises(ValueError, match="beta1"):
            gen.reconstruct(x, R, L, 0.01, z_init_val=z0, adam=(1.0, 0.999, 1e-8))
    finally:
        gen.close()


def test_defensegan_rec_optimizer_adam_is_the_native_adam_call():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp32")
    try:
        gan.rec_rr, gan.rec_iters, gan.rec_lr = 3, 8, 0.02
        gan.rec_optimizer, gan.rec_adam_betas, gan.rec_adam_eps = "adam", (0.8, 0.99), 1e-7
        x = torch.tensor(O.synthetic_images("mnist", gan.weights, 2)).cuda()
        z0 = _z0(6)
        got = gan.reconstruct(x, z_init_val=z0, return_aux=True)
        want = gan._native.reconstruct(x, 3, 8, 0.02, z_init_val=z0, adam=(0.8, 0.99, 1e-7), return_aux=True)
        assert _same([t.clone() for t in got], [t.clone() for t in want])
        a = torch.tensor(MO.block_average_operator(28, 28, 1, 2)).cuda()
        y = (x.reshape(2, -1).double() @ a.double().t()).float()
        got = gan.reconstruct_measured(y, a, z_init_val=z0, return_aux=True)
        want = gan._native.reconstruct_measured(y, a, 3, 8, 0.02, z_init_val=z0, adam=(0.8, 0.99, 1e-7), return_aux=True)
        assert _same([t.clone() for t in got], [t.clone() for t in want])
    finally:
        gan.close()
