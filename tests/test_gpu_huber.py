"""GPU tests (H100, -m gpu) of the Huber data term (dgan_reconstruct_huber, dgan_reconstruct_measured[_csr]_huber,
dgan_loss_grad[_measured[_csr]]_huber), on MNIST and CelebA, fp32 and fp16:
  - bit identities: delta = +inf gives the squared-error counterpart's rec, loss and idx bits on every entry (image,
    weighted, pruned, Adam, measured dense and CSR, BatchNorm), and delta = 2 on the image loss for in-range images; an
    identity prune schedule gives the unpruned Huber bits, any schedule the result composed from rec_rr = 1 calls; fp32
    CSR equals fp32 dense;
  - the loss of dgan_loss_grad[_measured[_csr]]_huber against fp64 from the G(z) the call returned, and the gradient
    against the Huber oracle, at several deltas;
  - each layer-direction of dgan_loss_grad_huber (weighted or not) and dgan_loss_grad_measured_huber against fp64 on the
    operands it read, read back from the workspace: the Huber last-layer forward's y, d(pre) and loss parts, and the
    stored Huber residual psi(r), the row loss and the adjoint product on it, at a delta that clips 20 - 80 % of the
    residuals (tests/huber_layer_ref.py); on an H100 80GB HBM3 (700 W) the largest error over its bound was 0.007 for
    d(pre) and 0.006 for the loss parts on the tensor cores, 0.021 for the fp32 d(pre), 0.061 for the stored residual,
    0.004 for the measured row loss and 0.16 for the adjoint product on the clipped residual;
  - R = 10, L = 200 against the fp64 Huber oracle (tests/huber_oracle.py): momentum per image within 1e-4, Adam within
    test_gpu_adam.py's bounds, image and measured loss, and the returned loss the Huber loss of the returned rec;
    on an H100 80GB HBM3 (700 W) the momentum arms were within 1.1e-8 (fp32) and 7.6e-7 (fp16) of the oracle, the Adam
    arms within 1.5e-5;
  - Huber and squared-error calls, and two deltas, alternating on one workspace give fresh handles' bits; the counts
    equal the counterpart's, and steady state allocates nothing;
  - a bad delta is refused before anything is enqueued; rec_huber_delta on DefenseGANBase is the native Huber call."""
import ctypes

import numpy as np
import pytest
import torch

import huber_oracle as H
import measured_oracle as MO
from gpu_support import bits as _bits, gen as _gen, images as _images, same as _same, z0 as _z0
from gpu_support import rec as _rec, rec_m as _rec_m, release_cached_memory  # noqa: F401
from gpu_support import layout, read_call, view, views
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}
ADAM = (0.9, 0.999, 1e-8)
CASES = [(p, a) for p in ("fp32", "fp16") for a in ("mnist", "celeba")]
INF = float("inf")


def _salt_and_pepper(x, arch, p, seed=5):
    """x with a share p of its pixels set to the ends of the generator's range at random."""
    g = torch.Generator().manual_seed(seed)
    lo = 0.0 if arch == "mnist" else -1.0
    hit = (torch.rand(x.shape, generator=g) < p).to(x.device)
    val = torch.where(torch.rand(x.shape, generator=g) < 0.5, lo, 1.0).to(x.device)
    return torch.where(hit, val, x)


# ---- bit identities ----

def _composed(gen, x, R, L, lr, z0, prune, measured=None, **kw):
    """The pruned call's result from rec_rr = 1 calls on the tiled images (or measurements)."""
    B = x.shape[0]
    xt = x.repeat_interleave(R, dim=0)
    if kw.get("pixel_weights") is not None:
        kw = dict(kw, pixel_weights=kw["pixel_weights"].repeat_interleave(R, dim=0))

    def call(n_it):
        if measured is not None:
            return _rec_m(gen, xt, measured, 1, n_it, lr, z0, **kw)
        return _rec(gen, xt, 1, n_it, lr, z0, **kw)
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
    B, R, L, lr = 4, 4, 12, 2.0
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        pw = torch.rand(x.shape, generator=torch.Generator().manual_seed(4)).cuda()
        # delta = +inf (and 2 on in-range images): the squared-error counterpart's bits on every image entry
        for kw in (dict(), dict(pixel_weights=pw), dict(prune=[(5, 2)]), dict(adam=ADAM),
                   dict(adam=ADAM, pixel_weights=pw, prune=[(3, 3), (7, 1)])):
            lr_k = 0.02 if "adam" in kw else lr
            sq = _rec(gen, x, R, L, lr_k, z0, **kw)
            assert bool(torch.isfinite(sq[1]).all())
            for delta in (INF, 2.0):
                assert _same(_rec(gen, x, R, L, lr_k, z0, huber_delta=delta, **kw), sq), (delta, kw)
        # a delta that clips: the identity schedule and the composed result
        xs = _salt_and_pepper(x, arch, 0.1)
        hub = _rec(gen, xs, R, L, lr, z0, huber_delta=0.1)
        assert not _same(hub, _rec(gen, xs, R, L, lr, z0))
        assert _same(_rec(gen, xs, R, L, lr, z0, huber_delta=0.1, prune=[(1, R), (6, R)]), hub)
        for kw in (dict(), dict(adam=ADAM, pixel_weights=pw)):
            lr_k = 0.02 if "adam" in kw else lr
            assert _same(_rec(gen, xs, R, L, lr_k, z0, huber_delta=0.1, prune=[(5, 2)], **kw),
                         _composed(gen, xs, R, L, lr_k, z0, [(5, 2)], huber_delta=0.1, **kw)), kw
        # the measured loss, dense and CSR
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (xs.reshape(B, -1).double() @ a.double().t()).float()
        acsr = a.to_sparse_csr()
        for op in (a, acsr):
            for kw in (dict(), dict(prune=[(5, 2)]), dict(adam=ADAM)):
                lr_k = 0.02 if "adam" in kw else lr
                assert _same(_rec_m(gen, y, op, R, L, lr_k, z0, huber_delta=INF, **kw), _rec_m(gen, y, op, R, L, lr_k, z0,
                                                                                               **kw)), kw
        mh = _rec_m(gen, y, a, R, L, lr, z0, huber_delta=0.05)
        assert bool(torch.isfinite(mh[1]).all()) and not _same(mh, _rec_m(gen, y, a, R, L, lr, z0))
        assert _same(_rec_m(gen, y, a, R, L, lr, z0, huber_delta=0.05, prune=[(1, R), (6, R)]), mh)
        assert _same(_rec_m(gen, y, a, R, L, lr, z0, huber_delta=0.05, prune=[(5, 2)]),
                     _composed(gen, y, R, L, lr, z0, [(5, 2)], measured=a, huber_delta=0.05))
        if precision == "fp32":
            assert _same(_rec_m(gen, y, acsr, R, L, lr, z0, huber_delta=0.05), mh)
            assert _same(_rec_m(gen, y, acsr, R, L, 0.02, z0, huber_delta=0.05, adam=ADAM, prune=[(5, 2)]),
                         _rec_m(gen, y, a, R, L, 0.02, z0, huber_delta=0.05, adam=ADAM, prune=[(5, 2)]))
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_bn_huber_runs_unpruned_and_refuses_a_schedule(precision):
    from defensegan_b200 import _native
    B, R, L = 3, 2, 6
    w, gen = _gen("mnist", precision, use_bn=True)
    try:
        x = _images("mnist", w, B)
        z0 = _z0(B * R)
        assert _same(_rec(gen, x, R, L, 2.0, z0, huber_delta=INF), _rec(gen, x, R, L, 2.0, z0))
        got = _rec(gen, _salt_and_pepper(x, "mnist", 0.1), R, L, 2.0, z0, huber_delta=0.1)
        assert bool(torch.isfinite(got[1]).all())
        ws, need = gen._workspace(B, R)
        prm = _native.dgan_rec_params(B, R, L, 2.0, 0.7, 0, 0, 0)
        sched = (_native.dgan_prune_point * 1)(_native.dgan_prune_point(2, 1))
        out = torch.empty_like(x)
        rc = gen.lib.dgan_reconstruct_huber(gen._handle, ctypes.byref(prm), None, 0.1, sched, 1, _native._ptr(x), None,
                                            _native._ptr(z0), _native._ptr(out), None, None, ws, need,
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == -3
    finally:
        gen.close()


# ---- loss_grad against fp64 ----

def _clip_share(d, delta):
    return float((d.abs() > delta).double().mean())


def _median_delta(d):
    """A delta that clips about half of the residuals d: their median magnitude, to two significant digits."""
    return float("%.2g" % float(d.abs().median()))


@pytest.mark.parametrize("precision,arch", CASES)
def test_loss_grad_entries_against_fp64(precision, arch):
    """The loss from the call's own G(z) in fp64 (fp32: to 1e-5; fp16: the G(z) the call returns is the epilogue's fp32
    y, so the same bound holds), and the gradient against the fp64 oracle (fp32: 1e-3, fp16: 5e-2 of its largest
    entry), weighted or not, dense and CSR, at several deltas."""
    B, R = 3, 2
    w, gen = _gen(arch, precision)
    try:
        x = _salt_and_pepper(_images(arch, w, B), arch, 0.1)
        z0 = _z0(B * R)
        pw = torch.rand(x.shape, generator=torch.Generator().manual_seed(4)).cuda()
        a = MO.gaussian_operator(300, int(np.prod(SHAPE[arch])), seed=1)
        ym = (x.reshape(B, -1).double().cpu().numpy() @ a.T.astype(np.float64)).astype(np.float32)
        ym = ym + np.random.RandomState(6).standard_normal(ym.shape).astype(np.float32) * 0.2
        at = torch.tensor(a).cuda()
        gtol = 1e-3 if precision == "fp32" else 5e-2
        y, _, _ = gen.loss_grad(x, z0, R)
        d_image = _median_delta(y.double() - x.double().repeat_interleave(R, dim=0))
        for delta in (d_image, 0.05, 1.0):
            for weights in (None, pw):
                y, loss, grad = gen.loss_grad(x, z0, R, pixel_weights=weights, huber_delta=delta)
                d = y.double() - x.double().repeat_interleave(R, dim=0)
                if delta == d_image:
                    share = _clip_share(d, delta)
                    assert 0.2 <= share <= 0.8, share
                wt = None if weights is None else weights.double().repeat_interleave(R, dim=0)
                ref = H.terms(d, delta, wt).mean(dim=(1, 2, 3))
                assert torch.allclose(loss.double(), ref, rtol=1e-5, atol=1e-7), (delta, weights is None)
                _, _, gref = H.loss_and_grad(arch, w, z0.cpu().numpy(), R, delta, images=x.cpu().numpy(),
                                             pixel_weights=None if weights is None else weights.cpu().numpy())
                err = float(np.abs(grad.cpu().numpy() - gref).max()) / max(float(np.abs(gref).max()), 1e-12)
                assert err <= gtol, (delta, weights is None, err)
        ymt = torch.tensor(ym).cuda().double().repeat_interleave(R, 0)
        g, _, _ = gen.loss_grad_measured(torch.tensor(ym).cuda(), at, z0, R)
        d_meas = _median_delta(g.reshape(B * R, -1).double() @ at.double().t() - ymt)
        for delta in (d_meas, 0.02, 1.0):
            outs = []
            for op in (at, at.to_sparse_csr()):
                g, loss, grad = gen.loss_grad_measured(torch.tensor(ym).cuda(), op, z0, R, huber_delta=delta)
                r = g.reshape(B * R, -1).double() @ at.double().t() - ymt
                if delta == d_meas:
                    share = _clip_share(r, delta)
                    assert 0.2 <= share <= 0.8, share
                ref = H.terms(r, delta).mean(dim=1)
                ltol = 1e-5 if precision == "fp32" or op.layout == torch.sparse_csr else 2e-3     # TF32 products
                assert torch.allclose(loss.double(), ref, rtol=ltol, atol=1e-7), (delta, op.layout)
                _, _, gref = H.loss_and_grad(arch, w, z0.cpu().numpy(), R, delta, operator=a, measurements=ym)
                err = float(np.abs(grad.cpu().numpy() - gref).max()) / max(float(np.abs(gref).max()), 1e-12)
                assert err <= gtol, (delta, op.layout, err)
                outs.append((g.clone(), loss.clone(), grad.clone()))
            if precision == "fp32":
                assert _same(outs[0], outs[1]), delta
    finally:
        gen.close()


# ---- against the fp64 oracle ----

# The Adam arms: test_gpu_adam.py's bounds - (max |loss_min - oracle| / max oracle loss_min, least share of images choosing
# the oracle's restart, bound on |rec - oracle| where they do).  The fp16 operands of 200 Adam steps pick among near-equal
# restarts, so Adam's loop is compared more loosely than momentum's; the momentum arms take the bar of the weighted and
# measured parity tests: per image |loss_min - oracle| <= 1e-4.
ADAM_TOL = {"fp32": (2e-3, 0.75, 2e-2), "fp16": (3e-2, 0.0, 1.5e-1)}


def _compare(precision, tag, rec, loss, idx, ref, adam):
    dl = np.abs(loss.cpu().numpy().astype(np.float64) - ref["loss_min"])
    agree = float((idx.cpu().numpy() == ref["idx"]).mean())
    print("%s %s: max|dloss| = %.3g (max loss %.3g), restart agreement %.2f"
          % (precision, tag, float(dl.max()), float(np.abs(ref["loss_min"]).max()), agree))
    if not adam:
        assert dl.max() <= 1e-4, tag
        return
    rel_tol, agree_min, rec_tol = ADAM_TOL[precision]
    assert float(dl.max()) / max(float(np.abs(ref["loss_min"]).max()), 1e-3) <= rel_tol, tag
    assert agree >= agree_min, tag
    same = idx.cpu().numpy() == ref["idx"]
    if same.any():
        d = np.abs(rec.cpu().numpy().reshape(ref["rec"].shape)[same] - ref["rec"][same]).max()
        assert d <= rec_tol, (tag, d)


@pytest.mark.parametrize("precision,arch", CASES)
def test_long_horizon_parity_with_the_fp64_oracle(precision, arch):
    """R = 10, L = 200 on images with 5 % salt-and-pepper pixels at delta = 0.1: momentum per image within 1e-4 of the
    fp64 oracle, Adam within test_gpu_adam.py's bounds; on every arm the returned loss is the Huber loss of the returned
    reconstruction (image loss: to 1e-6, the weighted test's bar; measured loss: test_gpu_measured.py's bar)."""
    B, R, L = (4, 10, 200) if arch == "mnist" else (2, 10, 200)
    delta = 0.1
    w, gen = _gen(arch, precision)
    try:
        imgs = _salt_and_pepper(torch.tensor(O.synthetic_images(arch, w, B)), arch, 0.05).numpy()
        z0 = O.sample_z0(B * R, 128)
        a = MO.block_average_operator(*SHAPE[arch], 2)
        ym = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
        at, xt, yt = torch.tensor(a).cuda(), torch.tensor(imgs).cuda(), torch.tensor(ym).cuda()
        for adam, lr in ((None, 10.0), (ADAM, 0.005)):
            kw = {} if adam is None else {"adam": adam}
            name = "adam" if adam else "momentum"
            ref = H.reconstruct(arch, w, R, L, lr, delta, images=imgs, z_init_val=z0, adam=adam, device="cuda")
            rec, loss, idx = _rec(gen, xt, R, L, lr, torch.tensor(z0).cuda(), huber_delta=delta, **kw)
            _compare(precision, "%s image %s" % (arch, name), rec, loss, idx, ref, adam is not None)
            hl = H.terms(rec.double() - xt.double(), delta).mean(dim=(1, 2, 3))
            assert float((hl - loss.double()).abs().max()) <= 1e-6, name
            ref = H.reconstruct(arch, w, R, L, lr, delta, operator=a, measurements=ym, z_init_val=z0, adam=adam,
                                device="cuda")
            for op, kind in ((at, "dense"), (at.to_sparse_csr(), "csr")):
                rec, loss, idx = _rec_m(gen, yt, op, R, L, lr, torch.tensor(z0).cuda(), huber_delta=delta, **kw)
                _compare(precision, "%s measured %s %s" % (arch, kind, name), rec, loss, idx, ref, adam is not None)
                ml = H.terms(rec.reshape(B, -1).double() @ at.double().t() - yt.double(), delta).mean(dim=1)
                # fp16 dense: the loss is that of the TF32 measurement product (test_gpu_measured.py's TOL)
                tol = 1e-4 if precision == "fp16" and kind == "dense" else 1e-5
                assert float((ml - loss.double()).abs().max()) <= tol * max(1.0, float(ml.abs().max())), (name, kind)
    finally:
        gen.close()


# ---- the Huber loss epilogues on their own operands, layer by layer ----

# (arch, latent_dim, net_dim, use_bn): test_gpu_weighted.py's matrix
LAYER_MATRIX = [("mnist", 128, 64, False), ("mnist", 128, 64, True), ("celeba", 128, 64, False), ("celeba", 64, 128, True)]


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("n_rows", [1, 2560])
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", LAYER_MATRIX)
def test_huber_loss_grad_each_layer_direction(arch, latent, net_dim, use_bn, precision, n_rows, weighted):
    """dgan_loss_grad_huber, weighted or not, read back from the workspace (the counterpart's layout): every forward
    layer-direction, the Huber last-layer forward (y, d(pre), loss parts: tests/huber_layer_ref.py) and every backward
    layer-direction, each against fp64 on the operands it read, at a delta (the median |y - x| of the squared-error call)
    that clips 20 - 80 % of the pixels, the share taken from the fp64 reference."""
    import huber_layer_ref as HR
    import layer_ref as LR
    w, gen = _gen(arch, precision, use_bn, latent, net_dim)
    try:
        R_ = 1 if n_rows == 1 else 2
        B = n_rows // R_
        imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=3, latent_dim=latent)).cuda()
        pw = torch.rand(imgs.shape, generator=torch.Generator().manual_seed(8)).cuda() if weighted else None
        z = torch.tensor(O.sample_z0(n_rows, latent, seed=4)).cuda()
        x_rows = imgs.reshape(B, -1).repeat_interleave(R_, dim=0)
        y, _, _ = gen.loss_grad(imgs, z, R_)
        delta = _median_delta(y.reshape(n_rows, -1).double() - x_rows.double())
        gen.loss_grad(imgs, z, R_, pixel_weights=pw, huber_delta=delta)
        torch.cuda.synchronize()
        w_rows = None if pw is None else pw.reshape(B, -1).repeat_interleave(R_, dim=0)
        ws, net = read_call(gen, w, arch, latent, net_dim, use_bn, precision, n_rows)
        stats = LR.Stats()
        LR.check_inputs(net, ws, n_rows, z)
        LR.check_forward(net, ws, n_rows, stats, "")
        share = HR.check_last_fwd_huber(net, ws, n_rows, x_rows, w_rows, delta, stats, "")
        LR.check_backward(net, ws, n_rows, stats, "")
        print("\nhuber %s %s latent=%d net_dim=%d bn=%d rows=%d weighted=%d delta=%g clipped=%.2f"
              % (precision, arch, latent, net_dim, use_bn, n_rows, weighted, delta, share))
        print("\n".join(stats.lines()))
        assert 0.2 <= share <= 0.8, share
    finally:
        gen.close()


@pytest.mark.parametrize("n_rows", [300, 2560])
@pytest.mark.parametrize("precision", ["fp16", "fp32"])
@pytest.mark.parametrize("arch,latent,net_dim,use_bn", LAYER_MATRIX)
def test_huber_loss_grad_measured_each_layer_direction(arch, latent, net_dim, use_bn, precision, n_rows):
    """dgan_loss_grad_measured_huber read back from the workspace: the forward, y, the stored Huber residual psi(r),
    the row loss and the adjoint product on it (tests/huber_layer_ref.py), the cotangent entry and the backward, each
    against fp64 on the operands it read, at a delta (the median |r| of the squared-error call) that clips 20 - 80 % of
    the residuals."""
    import huber_layer_ref as HR
    import layer_ref as LR
    w, gen = _gen(arch, precision, use_bn, latent, net_dim)
    try:
        R_ = 2
        B = n_rows // R_
        hwc = int(np.prod(SHAPE[arch]))
        m = 200 if arch == "mnist" else 1000
        imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=3, latent_dim=latent)).cuda()
        a = torch.tensor(MO.gaussian_operator(m, hwc, seed=m)).cuda()
        y = (imgs.reshape(B, -1).double() @ a.double().t()).float()
        z = torch.tensor(O.sample_z0(n_rows, latent, seed=4)).cuda()
        g, _, _ = gen.loss_grad_measured(y, a, z, R_)
        delta = _median_delta(g.reshape(n_rows, -1).double() @ a.double().t() - y.double().repeat_interleave(R_, 0))
        gen.loss_grad_measured(y, a, z, R_, huber_delta=delta)
        torch.cuda.synchronize()
        ws, net = read_call(gen, w, arch, latent, net_dim, use_bn, precision, n_rows)
        wsm = views(gen, layout(gen, "_measured", n_rows, m)[0][0])
        for k in ("am", "amt", "ym", "r", "dym", "mloss_part", "mscale"):
            ws[k] = wsm[k]
        stats = LR.Stats()
        LR.check_inputs(net, ws, n_rows, z)
        LR.check_forward(net, ws, n_rows, stats, "")
        LR.check_last_y(net, ws, n_rows, stats, "")
        share = HR.check_measured_huber(ws, n_rows, R_, m, hwc, delta, precision, stats, "")
        LR.check_cotangent(net, ws, n_rows, ws["dym"][:n_rows], stats, "", scale="mscale")
        LR.check_backward(net, ws, n_rows, stats, "")
        print("\nhuber measured %s %s latent=%d net_dim=%d bn=%d rows=%d m=%d delta=%g clipped=%.2f"
              % (precision, arch, latent, net_dim, use_bn, n_rows, m, delta, share))
        print("\n".join(stats.lines()))
        assert 0.2 <= share <= 0.8, share
    finally:
        gen.close()


# ---- calls on one handle, counts, steady state ----

@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_graph_cache_counts_and_steady_state(precision):
    arch, B, R, L = "mnist", 5, 3, 7
    w, gen = _gen(arch, precision)
    _, fresh = _gen(arch, precision)
    try:
        x = _salt_and_pepper(_images(arch, w, B), arch, 0.1)
        z0 = _z0(B * R)
        a = torch.tensor(MO.gaussian_operator(100, 784, seed=1)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()

        def call(g, kind):
            delta = {"sq": None, "h1": 0.1, "h2": 0.3, "hinf": INF}[kind[1:]]
            if kind[0] == "m":
                return _rec_m(g, y, a, R, L, 2.0, z0, huber_delta=delta)
            return _rec(g, x, R, L, 2.0, z0, huber_delta=delta)

        kinds = ("isq", "ih1", "ih2", "ihinf", "msq", "mh1", "mh2")
        want = {}
        for k in kinds:                                     # each on a fresh handle's first use of its key
            _, g = _gen(arch, precision)
            want[k] = call(g, k)
            g.close()
        assert not _same(want["ih1"], want["ih2"]) and not _same(want["isq"], want["ih1"])
        assert _same(want["ihinf"], want["isq"])
        for kind in ("ih1", "isq", "ih2", "ih1", "mh1", "msq", "mh2", "ihinf", "mh1", "isq", "ih2"):
            assert _same(call(gen, kind), want[kind]), kind
        for sq, hub in (("isq", "ih1"), ("msq", "mh1")):
            call(fresh, sq)
            enq, launches = fresh.last_enqueue_count, fresh.last_launch_count
            call(fresh, hub)
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            for _ in range(3):
                call(fresh, hub)
                assert (fresh.last_enqueue_count, fresh.last_launch_count) == (enq, launches), hub
            torch.cuda.synchronize()
            assert torch.cuda.mem_get_info()[0] == free0
        for kw in (dict(prune=[(3, 2)]), dict(adam=ADAM, pixel_weights=torch.ones_like(x), prune=[(2, 2), (5, 1)])):
            _rec(gen, x, R, L, 0.02, z0, **kw)
            counts = (gen.last_enqueue_count, gen.last_launch_count)
            _rec(gen, x, R, L, 0.02, z0, huber_delta=0.1, **kw)
            assert (gen.last_enqueue_count, gen.last_launch_count) == counts, kw
        _rec_m(gen, y, a.to_sparse_csr(), R, L, 0.02, z0, adam=ADAM, prune=[(3, 2)])
        counts = (gen.last_enqueue_count, gen.last_launch_count)
        _rec_m(gen, y, a.to_sparse_csr(), R, L, 0.02, z0, adam=ADAM, prune=[(3, 2)], huber_delta=0.1)
        assert (gen.last_enqueue_count, gen.last_launch_count) == counts
        # the workspace is the counterpart's: the same size, the same layout string (dgan_debug_workspace_layout
        # [_weighted]), and a Huber call leaves G(z) where that layout puts y
        for pw in (None, torch.ones_like(x)):
            regions, lay = layout(gen, "_weighted" if pw is not None else "", B * R)
            size = gen._workspace(B, R, weighted=pw is not None)[1]
            yh, _, _ = gen.loss_grad(x, z0, R, pixel_weights=pw, huber_delta=0.1)
            assert gen._workspace(B, R, weighted=pw is not None)[1] == size
            assert layout(gen, "_weighted" if pw is not None else "", B * R)[1] == lay
            stored = view(gen, regions[0], "y").flatten()[:B * R * 784].view(B * R, 784)
            assert torch.equal(_bits(stored), _bits(yh.reshape(B * R, 784)))
    finally:
        gen.close()
        fresh.close()


# ---- refusals and routing ----

def test_bad_delta_is_refused_before_anything_is_enqueued():
    from defensegan_b200 import _native
    B, R, L = 2, 2, 4
    w, gen = _gen("mnist", "fp32")
    try:
        x = _images("mnist", w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.block_average_operator(28, 28, 1, 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        prm = _native.dgan_rec_params(B, R, L, 2.0, 0.7, 0, 0, 0)
        out = torch.full_like(x, 7.0)
        loss = torch.full((B * R,), 7.0, device="cuda")
        grad = torch.full((B * R, 128), 7.0, device="cuda")
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = _native._ptr
        ws, need = gen._workspace(B, R)
        for bad in (0.0, -0.5, float("nan"), -INF):
            assert gen.lib.dgan_reconstruct_huber(gen._handle, ctypes.byref(prm), None, bad, None, 0, p(x), None, p(z0),
                                                  p(out), None, None, ws, need, stream) == -1
            assert b"Huber" in gen.lib.dgan_last_error()
            assert gen.lib.dgan_loss_grad_huber(gen._handle, bad, p(x), None, B, R, p(z0), None, p(loss), None, ws, need,
                                                stream) == -1
            wsm, needm = gen._workspace(B, R, m=a.shape[0])
            assert gen.lib.dgan_reconstruct_measured_huber(gen._handle, ctypes.byref(prm), None, bad, None, 0, p(a),
                                                           a.shape[0], p(y), p(z0), p(out), None, None, wsm, needm,
                                                           stream) == -1
            assert gen.lib.dgan_loss_grad_measured_huber(gen._handle, bad, p(a), a.shape[0], p(y), B, R, p(z0), None,
                                                         p(loss), p(grad), wsm, needm, stream) == -1
        # the counterpart's checks come first: a workspace too small is DGAN_ERR_WORKSPACE whatever the delta
        assert gen.lib.dgan_reconstruct_huber(gen._handle, ctypes.byref(prm), None, 0.0, None, 0, p(x), None, p(z0),
                                              p(out), None, None, ws, 1024, stream) == -4
        torch.cuda.synchronize()
        assert bool((out == 7.0).all()) and bool((loss == 7.0).all()) and bool((grad == 7.0).all())
        with pytest.raises(ValueError, match="huber_delta"):
            gen.reconstruct(x, R, L, 2.0, z_init_val=z0, huber_delta=0.0)
    finally:
        gen.close()


def test_defensegan_rec_huber_delta_is_the_native_huber_call():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp32")
    try:
        gan.rec_rr, gan.rec_iters, gan.rec_lr = 3, 8, 2.0
        gan.rec_huber_delta = 0.1
        x = _salt_and_pepper(torch.tensor(O.synthetic_images("mnist", gan.weights, 2)), "mnist", 0.1).cuda()
        z0 = _z0(6)
        got = gan.reconstruct(x, z_init_val=z0, return_aux=True)
        want = gan._native.reconstruct(x, 3, 8, 2.0, z_init_val=z0, huber_delta=0.1, return_aux=True)
        assert _same([t.clone() for t in got], [t.clone() for t in want])
        a = torch.tensor(MO.block_average_operator(28, 28, 1, 2)).cuda()
        y = (x.reshape(2, -1).double() @ a.double().t()).float()
        for op in (a, a.to_sparse_csr()):
            got = gan.reconstruct_measured(y, op, z_init_val=z0, return_aux=True)
            want = gan._native.reconstruct_measured(y, op, 3, 8, 2.0, z_init_val=z0, huber_delta=0.1, return_aux=True)
            assert _same([t.clone() for t in got], [t.clone() for t in want])
    finally:
        gan.close()
