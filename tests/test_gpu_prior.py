"""GPU tests (H100, -m gpu) of the latent prior (dgan_reconstruct_prior, dgan_reconstruct_measured[_csr / _conv]_prior),
J = D + lambda ||z||^2, on MNIST and CelebA, fp32 and fp16:
  - lambda = 0 gives the counterpart's rec, loss and idx bits on every entry: image, weighted, Huber, Adam, pruned, and
    measured dense, CSR and convolution (pruned and Adam too), and with BatchNorm unpruned;
  - at L = 1 the loop runs the forward only: the loss is D + lambda ||z0||^2 against fp64 on the call's own G(z0), and
    the restart follows J where the data term's arg-min differs;
  - the prior momentum and Adam updates against fp64 on the operands they read back from the workspace, steps k = 1, 2,
    with and without BatchNorm, image and measured loss;
  - R = 10, L = 200 against the fp64 prior oracle (tests/prior_oracle.py), image and measured loss;
  - pruning: keep = R gives the unpruned prior bits, a schedule the result composed from rec_rr = 1 prior calls, and a
    prune point ranks by J on the z of iteration iter_k - 1, not on the updated z;
  - the launch and enqueue counts of the header, the graph cache keyed on lambda, no allocation in steady state;
  - a bad lambda is refused before anything is enqueued; rec_z_prior on DefenseGANBase is the native prior call."""
import ctypes

import numpy as np
import pytest
import torch

import layer_ref as LR
import measured_oracle as MO
import prior_oracle as P
from gpu_support import bits as _bits, gen as _gen, images as _images, same as _same, z0 as _z0
from gpu_support import rec as _rec, rec_m as _rec_m, release_cached_memory  # noqa: F401
from gpu_support import gsum as _gsum, option_layout as _layout, option_lr as _lr, read as _read
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

HWC = {"mnist": 784, "celeba": 12288}
SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}
ADAM = (0.9, 0.999, 1e-8)
CASES = [(p, a) for p in ("fp32", "fp16") for a in ("mnist", "celeba")]


# ---- lambda = 0: the counterpart's bits ----

@pytest.mark.parametrize("precision,arch", CASES)
def test_lambda_zero_gives_the_counterparts_bits(precision, arch):
    from defensegan_b200.operators import ConvOperator
    B, R, L = 3, 4, 10
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        pw = torch.rand(x.shape, generator=torch.Generator().manual_seed(4)).cuda()
        for kw in (dict(), dict(pixel_weights=pw), dict(huber_delta=0.1), dict(adam=ADAM), dict(prune=[(5, 2)]),
                   dict(adam=ADAM, pixel_weights=pw, prune=[(3, 3), (7, 1)]), dict(huber_delta=0.1, prune=[(4, 2)])):
            want = _rec(gen, x, R, L, _lr(kw), z0, **kw)
            assert bool(torch.isfinite(want[1]).all())
            assert _same(_rec(gen, x, R, L, _lr(kw), z0, z_prior=0.0, **kw), want), kw
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        conv = ConvOperator.box(2)
        yc = conv(x.double()).float()
        for op, ym in ((a, y), (a.to_sparse_csr(), y), (conv, yc)):
            for kw in (dict(), dict(prune=[(5, 2)]), dict(adam=ADAM), dict(adam=ADAM, prune=[(2, 3), (6, 1)]),
                       dict(huber_delta=0.05)):
                want = _rec_m(gen, ym, op, R, L, _lr(kw), z0, **kw)
                assert bool(torch.isfinite(want[1]).all())
                assert _same(_rec_m(gen, ym, op, R, L, _lr(kw), z0, z_prior=0.0, **kw), want), (type(op), kw)
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_bn_prior_runs_unpruned_and_refuses_a_schedule(precision):
    from defensegan_b200 import _native
    B, R, L = 3, 2, 6
    w, gen = _gen("mnist", precision, use_bn=True)
    try:
        x = _images("mnist", w, B)
        z0 = _z0(B * R)
        for kw in (dict(), dict(adam=ADAM)):
            assert _same(_rec(gen, x, R, L, _lr(kw), z0, z_prior=0.0, **kw), _rec(gen, x, R, L, _lr(kw), z0, **kw))
            got = _rec(gen, x, R, L, _lr(kw), z0, z_prior=0.1, **kw)
            assert bool(torch.isfinite(got[1]).all())
        ws, need = gen._workspace(B, R)
        prm = _native.dgan_rec_params(B, R, L, 0.5, 0.7, 0, 0, 0)
        sched = (_native.dgan_prune_point * 1)(_native.dgan_prune_point(2, 1))
        out = torch.empty_like(x)
        rc = gen.lib.dgan_reconstruct_prior(gen._handle, ctypes.byref(prm), None, None, 0.1, sched, 1, _native._ptr(x),
                                            None, _native._ptr(z0), _native._ptr(out), None, None, ws, need,
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == -3
    finally:
        gen.close()


# ---- the objective at L = 1 ----

@pytest.mark.parametrize("precision,arch", CASES)
def test_objective_at_one_step_follows_j(precision, arch):
    """Restart 0 is the latent the image was generated from (D about 0, ||z||^2 about 9), restart 1 a short random latent
    (D clearly larger, ||z||^2 about 0.09): the data term picks restart 0, J at lambda = 1 restart 1.  L = 1 runs the
    forward only, so the loss is D + lambda ||z0||^2 of the chosen restart, against fp64 on the returned G(z0)."""
    B, R, lam = 4, 2, 1.0
    w, gen = _gen(arch, precision)
    try:
        zt = _z0(B, seed=8)
        zt = zt * (3.0 / zt.norm(dim=1, keepdim=True))
        x = gen.forward(zt).reshape((B,) + SHAPE[arch]).contiguous()
        zr = _z0(B, seed=9)
        zr = zr * (0.3 / zr.norm(dim=1, keepdim=True))
        z0 = torch.stack([zt, zr], dim=1).reshape(B * R, -1).contiguous()
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()

        def data(rec):
            return ((rec.double() - x.double()) ** 2).reshape(B, -1).mean(dim=1)

        def mdata(rec):
            return ((rec.reshape(B, -1).double() @ a.double().t() - y.double()) ** 2).mean(dim=1)

        for call, dfn, tol in ((lambda **kw: _rec(gen, x, R, 1, 0.5, z0, **kw), data, 1e-6),
                               (lambda **kw: _rec_m(gen, y, a, R, 1, 0.5, z0, **kw), mdata,
                                1e-4 if precision == "fp16" else 1e-6)):
            rec0, loss0, idx0 = call()
            assert idx0.tolist() == [0] * B
            rec, loss, idx = call(z_prior=lam)
            assert idx.tolist() == [1] * B
            zc = z0.reshape(B, R, -1)[torch.arange(B), idx.long()].double()
            want = dfn(rec) + lam * (zc * zc).sum(dim=1)
            assert float((loss.double() - want).abs().max()) <= tol * max(1.0, float(want.abs().max()))
            # the prior term is the fp32 fmaf chain over the real columns, added once to the finished data term
            zf = zc.float()
            acc = torch.zeros(B, dtype=torch.float32, device="cuda")
            for j in range(zf.shape[1]):
                acc = torch.addcmul(acc, zf[:, j], zf[:, j])
            assert float((loss.double() - dfn(rec) - acc.double() * lam).abs().max()) <= tol * 2
    finally:
        gen.close()


# ---- the update on its stored operands ----

def _check_steps(ws_list, z0p, lr, lam, n, lat, tc, row_mul, pad_rows_zero, tag, adam=None, mu=0.7):
    """ws_list[k - 1] after L = k + 1 (step k) from the same z0: v (m), s and z against fp64 of the prior update on the
    operands the kernel read - the stored split-K parts times the multiplier, plus 2 lambda times the previous step's
    stored z - to a few fp32 ulps of the magnitudes of their terms.  Padded latent channels exactly 0 (and,
    pad_rows_zero, the tile-padding rows); z_h = RN16(z)."""
    tl = float(np.float32(2 * np.float32(lam)))
    prev = dict(v=torch.zeros_like(ws_list[0]["v"]).double(), s=torch.zeros_like(ws_list[0]["v"]).double(),
                z=z0p.double())
    for k, ws in enumerate(ws_list, 1):
        gd = (_gsum(ws["g"]) * row_mul).double()
        gp = gd + tl * prev["z"]
        gabs = gd.abs() + tl * prev["z"].abs()
        if adam is None:
            v_ref = mu * prev["v"] + gp
            v_abs = mu * prev["v"].abs() + gabs
            u_ref = lr * ws["v"].double()
            checks = [("v", ws["v"], v_ref, 4 * LR.half_ulp(v_abs, "f32"))]
        else:
            b1, b2, eps = (float(np.float32(t)) for t in adam)
            import adam_oracle as AO
            c1, c2 = AO.adam_constants(lr, k - 1, b1, b2)
            v_ref = b1 * prev["v"] + (1 - b1) * gp
            v_abs = b1 * prev["v"].abs() + (1 - b1) * gabs
            s_ref = b2 * prev["s"] + (1 - b2) * gp * gp
            s_abs = b2 * prev["s"] + (1 - b2) * gabs * gabs
            u_ref = c1 * ws["v"].double() / (torch.sqrt(ws["s"].double()) * c2 + eps)
            checks = [("m", ws["v"], v_ref, 4 * LR.half_ulp(v_abs, "f32")),
                      ("s", ws["s"], s_ref, 8 * LR.half_ulp(s_abs, "f32"))]
        z_ref = prev["z"] - u_ref
        checks.append(("z", ws["z"], z_ref, 2 * LR.half_ulp(prev["z"], "f32") + 12 * LR.half_ulp(u_ref, "f32")))
        for name, got, ref, bound in checks:
            err = (got.double() - ref).abs()
            bound = bound + 2.0 ** -149
            assert bool((err <= bound).all()), "%s k=%d %s: max err / bound %.3g" % (tag, k, name,
                                                                                     float((err / bound).max()))
            if pad_rows_zero:
                LR.check_pad_rows_zero("%s k=%d %s" % (tag, k, name), got, n)
            LR.check_zero_pad("%s k=%d %s" % (tag, k, name), got, lat)
        if tc:
            assert torch.equal(ws["z_h"], ws["z"].half()), "%s k=%d: z_h is not RN16(z)" % (tag, k)
        prev = dict(v=ws["v"].double(), s=ws["s"].double() if adam else prev["s"], z=ws["z"].double())


@pytest.mark.parametrize("use_bn", [False, True])
@pytest.mark.parametrize("precision,arch", CASES)
def test_update_on_its_stored_operands(precision, arch, use_bn):
    lat, B, R, lam = 100, 3, 2, 0.3
    w, gen = _gen(arch, precision, use_bn=use_bn, latent=lat)
    tc = precision == "fp16"
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R, lat)
        gmul = torch.tensor(2.0, dtype=torch.float32) / torch.tensor(float(HWC[arch]), dtype=torch.float32)
        if tc:
            gmul = gmul / torch.tensor(LR.GRAD_SCALE, dtype=torch.float32)
        a = torch.tensor(MO.gaussian_operator(64, HWC[arch], seed=1)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        for adam, lr in ((None, 0.5), (ADAM, 0.01)):
            kw = {} if adam is None else {"adam": adam}
            names = ("g", "v", "z") + (("s",) if adam else ()) + (("z_h",) if tc else ())
            bufs, _ = _layout(gen, B, R, adam=adam is not None)
            out = []
            for L in (2, 3):
                _rec(gen, x, R, L, lr, z0, z_prior=lam, **kw)
                out.append({nm: _read(gen, bufs, nm) for nm in names})
            z0p = torch.zeros_like(out[0]["z"])
            z0p[:B * R, :lat] = z0
            # the fp16 image loss's last-layer forward leaves a gradient in the tile-padding rows, as without the prior
            tag = "%s %s image %s" % (precision, arch, "adam" if adam else "momentum")
            _check_steps(out, z0p, lr, lam, B * R, lat, tc, gmul.item(), not tc, tag, adam)
            if use_bn:
                continue
            bufs, _ = _layout(gen, B, R, m=64, adam=adam is not None)
            out = []
            for L in (2, 3):
                _rec_m(gen, y, a, R, L, lr, z0, z_prior=lam, **kw)
                out.append({nm: _read(gen, bufs, nm) for nm in names + ("mscale",)})
            for o in out:
                scale = torch.ones(o["z"].shape[0], 1, device="cuda")
                if tc:
                    scale[:B * R, 0] = 1.0 / o["mscale"][:B * R]
                o["g"] = o["g"] * scale.unsqueeze(0)                 # exact: power-of-two scales
            tag = "%s %s measured %s" % (precision, arch, "adam" if adam else "momentum")
            _check_steps(out, z0p, lr, lam, B * R, lat, tc, 1.0, True, tag, adam)
    finally:
        gen.close()


# ---- against the fp64 oracle ----

# Adam: test_gpu_adam.py's bounds (relative loss, rec where the restarts agree); momentum: the Huber parity test's 1e-4
# per image on the loss.  The prior pulls the restarts of an image to one optimum, so the restart index is a tie-break
# among near-equal values: instead of the restart agreement, the oracle's J of the restart the library chose must be the
# oracle's minimum to the loss tolerance.  On an H100 80GB HBM3 (700 W) the losses were within 1.3e-9 (fp32) and 7.8e-7
# (fp16) of the oracle's, and the oracle's J of the chosen restart within 3.4e-10 of its minimum.
ADAM_TOL = {"fp32": (2e-3, 2e-2), "fp16": (3e-2, 1.5e-1)}


def _compare(precision, tag, rec, loss, idx, ref, adam, R):
    dl = np.abs(loss.cpu().numpy().astype(np.float64) - ref["loss_min"])
    idx_np = idx.cpu().numpy()
    chosen = ref["loss_all"][np.arange(len(idx_np)) * R + idx_np]
    agree = float((idx_np == ref["idx"]).mean())
    scale = max(float(np.abs(ref["loss_min"]).max()), 1e-3)
    print("%s %s: max|dloss| = %.3g (max loss %.3g), restart agreement %.2f, max oracle J(chosen) - min %.3g"
          % (precision, tag, float(dl.max()), scale, agree, float((chosen - ref["loss_min"]).max())))
    tol = 1e-4 if not adam else ADAM_TOL[precision][0] * scale
    assert dl.max() <= tol, tag
    assert float((chosen - ref["loss_min"]).max()) <= tol, tag
    if adam:
        same = idx_np == ref["idx"]
        if same.any():
            d = np.abs(rec.cpu().numpy().reshape(ref["rec"].shape)[same] - ref["rec"][same]).max()
            assert d <= ADAM_TOL[precision][1], (tag, d)


@pytest.mark.parametrize("precision,arch", CASES)
def test_long_horizon_parity_with_the_fp64_oracle(precision, arch):
    """R = 10, L = 200: momentum at lambda = 0.01 (rec_lr 10) and Adam at lambda = 0.1 (rec_lr 0.005), image loss and
    2x2 block-average measurements (dense and CSR)."""
    B, R, L = (4, 10, 200) if arch == "mnist" else (2, 10, 200)
    w, gen = _gen(arch, precision)
    try:
        imgs = O.synthetic_images(arch, w, B)
        z0 = O.sample_z0(B * R, 128)
        a = MO.block_average_operator(*SHAPE[arch], 2)
        ym = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
        at, xt, yt, z0t = torch.tensor(a).cuda(), torch.tensor(imgs).cuda(), torch.tensor(ym).cuda(), torch.tensor(z0).cuda()
        for adam, lr, lam in ((None, 10.0, 0.01), (ADAM, 0.005, 0.1)):
            kw = {} if adam is None else {"adam": adam}
            name = "adam" if adam else "momentum"
            ref = P.reconstruct(arch, w, R, L, lr, lam, images=imgs, z_init_val=z0, adam=adam, device="cuda")
            rec, loss, idx = _rec(gen, xt, R, L, lr, z0t, z_prior=lam, **kw)
            _compare(precision, "%s image %s" % (arch, name), rec, loss, idx, ref, adam is not None, R)
            ref = P.reconstruct(arch, w, R, L, lr, lam, operator=a, measurements=ym, z_init_val=z0, adam=adam,
                                device="cuda")
            for op, kind in ((at, "dense"), (at.to_sparse_csr(), "csr")):
                rec, loss, idx = _rec_m(gen, yt, op, R, L, lr, z0t, z_prior=lam, **kw)
                _compare(precision, "%s measured %s %s" % (arch, kind, name), rec, loss, idx, ref,
                         adam is not None, R)
    finally:
        gen.close()


# ---- pruning ----

def _composed(gen, x, R, L, lr, z0, prune, measured=None, **kw):
    """The pruned call's result from rec_rr = 1 calls on the tiled images (or measurements)."""
    B = x.shape[0]
    xt = x.repeat_interleave(R, dim=0)

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
def test_pruning_bit_identities(precision, arch):
    B, R, L, lam = 4, 4, 12, 0.05
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.block_average_operator(*SHAPE[arch], 2)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        for kw in (dict(), dict(adam=ADAM), dict(huber_delta=0.1)):
            plain = _rec(gen, x, R, L, _lr(kw), z0, z_prior=lam, **kw)
            assert bool(torch.isfinite(plain[1]).all())
            assert not _same(plain, _rec(gen, x, R, L, _lr(kw), z0, **kw)), kw
            for sched in ([(5, R)], [(1, R), (6, R), (11, R)]):
                assert _same(_rec(gen, x, R, L, _lr(kw), z0, z_prior=lam, prune=sched, **kw), plain), (sched, kw)
            for sched in ([(5, 2)], [(3, 3), (6, 2), (9, 1)]):
                assert _same(_rec(gen, x, R, L, _lr(kw), z0, z_prior=lam, prune=sched, **kw),
                             _composed(gen, x, R, L, _lr(kw), z0, sched, z_prior=lam, **kw)), (sched, kw)
            mplain = _rec_m(gen, y, a, R, L, _lr(kw), z0, z_prior=lam, **kw)
            assert _same(_rec_m(gen, y, a, R, L, _lr(kw), z0, z_prior=lam, prune=[(1, R), (6, R)], **kw), mplain), kw
            assert _same(_rec_m(gen, y, a, R, L, _lr(kw), z0, z_prior=lam, prune=[(5, 2)], **kw),
                         _composed(gen, y, R, L, _lr(kw), z0, [(5, 2)], measured=a, z_prior=lam, **kw)), kw
    finally:
        gen.close()


@pytest.mark.parametrize("precision,arch", CASES)
def test_prune_point_ranks_by_j_before_the_update(precision, arch):
    """Two restarts per image, lambda = 10, Adam (rec_lr 0.5), one prune point at iteration 1 keeping 1.  Restart 0 has
    every coordinate at magnitude 1 (||z||^2 = d); restart 1 half at sqrt(1.9), half at sqrt(0.05) (||z||^2 = 0.975 d),
    so J at iteration 0 ranks restart 1 first by 0.025 lambda d, far more than the data terms differ.  Adam's first
    step moves every coordinate by rec_lr towards 0 (2 lambda z dominates the data gradient), which leaves restart 0
    at 0.25 d and restart 1 at about 0.42 d: ranking with the updated z would keep restart 0."""
    B, R, L, lam, lr = 3, 2, 2, 10.0, 0.5
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        d = 128
        sign = torch.where(torch.rand(B * R, d, generator=torch.Generator().manual_seed(6)) < 0.5, -1.0, 1.0)
        mag = torch.ones(B * R, d)
        mag[1::R, : d // 2] = 1.9 ** 0.5
        mag[1::R, d // 2:] = 0.05 ** 0.5
        z0 = (sign * mag).cuda().contiguous()
        # the premise, in fp64 on the data terms and gradients the library computes at z0
        _, dl, g = gen.loss_grad(x, z0, R)
        dl, g, zd = dl.double().reshape(B, R), g.double(), z0.double()
        gp = g + 2 * lam * zd
        z1 = zd - lr * torch.sign(gp)                        # Adam's first step: c1 m / (sqrt(s) c2 + eps) = lr sign(g')
        j0 = dl + lam * (zd * zd).sum(dim=1).reshape(B, R)
        j1 = dl + lam * (z1 * z1).sum(dim=1).reshape(B, R)
        assert j0.argmin(dim=1).tolist() == [1] * B and j1.argmin(dim=1).tolist() == [0] * B
        rec, loss, idx = _rec(gen, x, R, L, lr, z0, adam=ADAM, z_prior=lam, prune=[(1, 1)])
        assert idx.tolist() == [1] * B
        # the survivor then runs alone: its result is that of restart 1 in a call of its own
        single = _rec(gen, x, 1, L, lr, z0[1::R].contiguous(), adam=ADAM, z_prior=lam)
        assert _same([rec, loss], single[:2])
    finally:
        gen.close()


# ---- counts, cache, steady state ----

@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_graph_cache_counts_and_steady_state(precision):
    from defensegan_b200.operators import ConvOperator
    arch, B, R, L = "mnist", 5, 3, 7
    w, gen = _gen(arch, precision)
    try:
        x = _images(arch, w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.gaussian_operator(100, 784, seed=1)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float()
        conv = ConvOperator.box(4)
        yc = conv(x.double()).float()
        extra_mom = (L - 1) if precision == "fp16" else 0
        cases = [("image momentum", lambda **kw: _rec(gen, x, R, L, 0.5, z0, **kw), extra_mom, 0),
                 ("image adam", lambda **kw: _rec(gen, x, R, L, 0.02, z0, adam=ADAM, **kw), 0, 0),
                 ("weighted", lambda **kw: _rec(gen, x, R, L, 0.5, z0, pixel_weights=torch.ones_like(x), **kw),
                  extra_mom, 0),
                 ("pruned", lambda **kw: _rec(gen, x, R, L, 0.5, z0, prune=[(2, 2), (5, 1)], **kw), extra_mom, 2),
                 ("measured", lambda **kw: _rec_m(gen, y, a, R, L, 0.5, z0, **kw), 0, 0),
                 ("csr pruned adam", lambda **kw: _rec_m(gen, y, a.to_sparse_csr(), R, L, 0.02, z0, adam=ADAM,
                                                         prune=[(3, 2)], **kw), 0, 1),
                 ("conv huber", lambda **kw: _rec_m(gen, yc, conv, R, L, 0.5, z0, huber_delta=0.1, **kw), 0, 0)]
        for name, call, extra, n_points in cases:
            call()
            enq, launches = gen.last_enqueue_count, gen.last_launch_count
            call(z_prior=0.1)
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            for _ in range(2):
                call(z_prior=0.1)
                assert gen.last_enqueue_count == enq, name
                assert gen.last_launch_count == launches + 1 + n_points + extra, name
            torch.cuda.synchronize()
            assert torch.cuda.mem_get_info()[0] == free0, name
        # the cache keys on lambda: each lambda gives a fresh handle's bits, alternating on one workspace
        want = {}
        for lam in (None, 0.0, 0.1, 0.3):
            _, g = _gen(arch, precision)
            want[lam] = _rec(g, x, R, L, 0.5, z0, z_prior=lam)
            g.close()
        assert _same(want[None], want[0.0]) and not _same(want[0.1], want[0.3]) and not _same(want[0.0], want[0.1])
        for lam in (0.1, 0.3, None, 0.1, 0.0, 0.3):
            assert _same(_rec(gen, x, R, L, 0.5, z0, z_prior=lam), want[lam]), lam
    finally:
        gen.close()


# ---- refusals and routing ----

def test_bad_lambda_is_refused_before_anything_is_enqueued():
    from defensegan_b200 import _native
    from defensegan_b200.operators import ConvOperator
    B, R, L = 2, 2, 4
    w, gen = _gen("mnist", "fp32")
    try:
        x = _images("mnist", w, B)
        z0 = _z0(B * R)
        a = torch.tensor(MO.gaussian_operator(50, 784, seed=1)).cuda()
        y = (x.reshape(B, -1).double() @ a.double().t()).float().contiguous()
        acsr = a.to_sparse_csr()
        rp, ci = acsr.crow_indices().int().contiguous(), acsr.col_indices().int().contiguous()
        val = acsr.values().contiguous()
        conv = ConvOperator.box(4)
        yc = conv(x.double()).float().reshape(B, -1).contiguous()
        k = conv.kernels(B, x.device).contiguous()
        op = _native.dgan_conv_op(4, 4, 0, 0, 4)
        _rec(gen, x, R, L, 0.5, z0)
        prm = _native.dgan_rec_params(B, R, L, 0.5, 0.7, 0, 0, 0)
        out = torch.full_like(x, 7.0)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = _native._ptr
        nnz = int(val.numel())
        ws = lambda **kw: gen._workspace(B, R, **kw)      # noqa: E731  (taken right before each call: it may grow)
        calls = {
            "image": lambda lam: gen.lib.dgan_reconstruct_prior(gen._handle, ctypes.byref(prm), None, None, lam, None, 0,
                                                                p(x), None, p(z0), p(out), None, None, *ws(), stream),
            "dense": lambda lam: gen.lib.dgan_reconstruct_measured_prior(gen._handle, ctypes.byref(prm), None, None, lam,
                                                                         None, 0, p(a), 50, p(y), p(z0), p(out), None,
                                                                         None, *ws(m=50), stream),
            "csr": lambda lam: gen.lib.dgan_reconstruct_measured_csr_prior(gen._handle, ctypes.byref(prm), None, None, lam,
                                                                           None, 0, p(rp), p(ci), p(val), 50, nnz, p(y),
                                                                           p(z0), p(out), None, None,
                                                                           *ws(m=50, nnz=nnz), stream),
            "conv": lambda lam: gen.lib.dgan_reconstruct_measured_conv_prior(gen._handle, ctypes.byref(prm), None, None,
                                                                             lam, None, 0, ctypes.byref(op), p(k), p(yc),
                                                                             p(z0), p(out), None, None, *ws(conv=op),
                                                                             stream)}
        for kind, call in calls.items():
            for bad in (float("nan"), float("inf"), -float("inf"), -0.5, 2e38):
                before = (gen.last_enqueue_count, gen.last_launch_count)
                assert call(bad) == -1, (kind, bad)
                assert b"z_prior" in gen.lib.dgan_last_error(), (kind, bad)
                assert (gen.last_enqueue_count, gen.last_launch_count) == before, (kind, bad)
        torch.cuda.synchronize()
        assert bool((out == 7.0).all())
        for bad in (float("nan"), -1.0, 2e38):
            with pytest.raises(ValueError, match="z_prior"):
                gen.reconstruct(x, R, L, 0.5, z_init_val=z0, z_prior=bad)
            with pytest.raises(ValueError, match="z_prior"):
                gen.reconstruct_measured(y, a, R, L, 0.5, z_init_val=z0, z_prior=bad)
    finally:
        gen.close()


def test_defensegan_rec_z_prior_is_the_native_prior_call():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp32")
    try:
        gan.rec_rr, gan.rec_iters, gan.rec_lr = 3, 8, 0.5
        gan.rec_z_prior = 0.2
        x = torch.tensor(O.synthetic_images("mnist", gan.weights, 2)).cuda()
        z0 = _z0(6)
        got = gan.reconstruct(x, z_init_val=z0, return_aux=True)
        want = gan._native.reconstruct(x, 3, 8, 0.5, z_init_val=z0, z_prior=0.2, return_aux=True)
        assert _same([t.clone() for t in got], [t.clone() for t in want])
        assert not _same([t.clone() for t in got], _rec(gan._native, x, 3, 8, 0.5, z0))
        a = torch.tensor(MO.block_average_operator(28, 28, 1, 2)).cuda()
        y = (x.reshape(2, -1).double() @ a.double().t()).float()
        got = gan.reconstruct_measured(y, a, z_init_val=z0, return_aux=True)
        want = gan._native.reconstruct_measured(y, a, 3, 8, 0.5, z_init_val=z0, z_prior=0.2, return_aux=True)
        assert _same([t.clone() for t in got], [t.clone() for t in want])
    finally:
        gan.close()
