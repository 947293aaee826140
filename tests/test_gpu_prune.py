"""GPU tests (H100, -m gpu) of restart pruning (dgan_reconstruct_pruned), on MNIST and CelebA, fp32 and fp16, unweighted
and weighted:
  - an identity schedule (keep = R at every point) gives the plain call's bits (rec, loss, idx), with decay_lr on and off;
  - one- and three-point schedules give the bits of the result composed from rec_rr = 1 plain calls on the tiled images
    (rows are independent without BatchNorm): each row's loss at iteration iter_k - 1, its final reconstruction and
    loss, then the ranking rule of the header;
  - ties (duplicated z0 rows) keep the lower original index; an image with a NaN pixel keeps restarts 0 .. keep-1 and
    returns idx 0;
  - batch-split invariance (the sharded call's semantics), and a seeded z0 equal to passing sample_z0's draw;
  - the gathered z / v (/ z_h) rows read back from the next region equal the source rows under the map;
  - the documented launch and enqueue counts, a replayed graph and no allocation in steady state;
  - DGAN_ERR_INVALID_ARG / DGAN_ERR_UNSUPPORTED / DGAN_ERR_WORKSPACE leave rec_dev untouched."""
import ctypes

import numpy as np
import pytest
import torch

from gpu_support import bits as _bits, gen as _gen, layout, read as _read, same as _same, ws_base
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

CASES = [(p, a, wt) for p in ("fp32", "fp16") for a in ("mnist", "celeba") for wt in (False, True)]
ONE = [(5, 2)]
THREE = [(3, 3), (6, 2), (9, 1)]


def _problem(arch, w, B, R, seed=2):
    x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=seed)).cuda()
    z0 = torch.tensor(O.sample_z0(B * R, 128, seed=seed + 1)).cuda()
    pw = torch.tensor(np.random.RandomState(seed).uniform(0, 1, size=tuple(x.shape)).astype(np.float32)).cuda()
    return x, z0, pw


def _call(gen, x, R, L, z0, pw, prune, lr=10.0, decay=False, **kw):
    return [t.clone() for t in gen.reconstruct(x, R, L, lr, z_init_val=z0, pixel_weights=pw, prune=prune, decay_lr=decay,
                                               return_aux=True, **kw)]


def _before(a, b):
    """prune_before of kernels_prune.cuh on (loss, original index) pairs."""
    (la, oa), (lb, ob) = a, b
    na, nb = np.isnan(la), np.isnan(lb)
    if na or nb:
        return (nb and oa < ob) if na else True
    return la < lb or (la == lb and oa < ob)


def _composed(gen, x, R, L, z0, pw, prune):
    """The pruned call's result from rec_rr = 1 plain calls on the tiled images (decay_lr off)."""
    B = x.shape[0]
    xt = x.repeat_interleave(R, dim=0)
    pt = pw.repeat_interleave(R, dim=0) if pw is not None else None
    loss_at = {}
    for it, _ in prune:
        loss_at[it] = _call(gen, xt, 1, it, z0, pt, None)[1].cpu().numpy()
    rec_all, loss_all, _ = _call(gen, xt, 1, L, z0, pt, None)
    loss_all = loss_all.cpu().numpy()
    rec, loss, idx = torch.empty_like(x), torch.empty(B, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda")
    for i in range(B):
        alive = list(range(R))
        for it, keep in prune:
            ranked = [(float(loss_at[it][i * R + r]), r) for r in alive]
            kept = [p for p in ranked if sum(_before(q, p) for q in ranked) < keep]
            alive = sorted(r for _, r in kept)
        best = alive[0]
        for r in alive[1:]:
            if loss_all[i * R + r] < loss_all[i * R + best]:
                best = r
        rec[i] = rec_all[i * R + best]
        loss[i] = float(loss_all[i * R + best])
        idx[i] = best
    return [rec, loss, idx]


@pytest.mark.parametrize("decay", [False, True])
@pytest.mark.parametrize("precision,arch,weighted", CASES)
def test_identity_schedule_gives_the_plain_bits(precision, arch, weighted, decay):
    w, gen = _gen(arch, precision)
    try:
        B, R, L = 3, 4, 12
        x, z0, pw = _problem(arch, w, B, R)
        pw = pw if weighted else None
        plain = _call(gen, x, R, L, z0, pw, None, decay=decay)
        for sched in ([(5, R)], [(1, R), (6, R), (11, R)]):
            assert _same(_call(gen, x, R, L, z0, pw, sched, decay=decay), plain), sched
    finally:
        gen.close()


@pytest.mark.parametrize("sched", [ONE, THREE], ids=["one", "three"])
@pytest.mark.parametrize("precision,arch,weighted", CASES)
def test_pruned_call_equals_the_composed_result(precision, arch, weighted, sched):
    w, gen = _gen(arch, precision)
    try:
        B, R, L = 5, 4, 12
        x, z0, pw = _problem(arch, w, B, R)
        pw = pw if weighted else None
        got = _call(gen, x, R, L, z0, pw, sched)
        want = _composed(gen, x, R, L, z0, pw, sched)
        assert _same(got, want)
        assert int(got[2].min()) >= 0 and int(got[2].max()) < R
        plain = _call(gen, x, R, L, z0, pw, None)
        print("\n%s %s weighted=%d %s: restart agreement with the unpruned call %.2f" % (
            precision, arch, weighted, sched, float((plain[2] == got[2]).float().mean())))
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_ties_keep_the_lower_index_and_nan_images_keep_restart_0(precision):
    arch, B, R, L = "mnist", 3, 4, 10
    w, gen = _gen(arch, precision)
    try:
        x, z0, _ = _problem(arch, w, B, R)
        z0[1:R] = z0[0]                                  # image 0: four identical restarts, identical losses
        x[2, 3, 4, 0] = float("nan")                     # image 2: every loss NaN
        for sched in ([(4, 2)], [(2, 3), (6, 1)]):
            got = _call(gen, x, R, L, z0, None, sched)
            assert _same(got, _composed(gen, x, R, L, z0, None, sched)), sched
            assert int(got[2][0]) == 0 and int(got[2][2]) == 0, sched
            assert bool(torch.isnan(got[1][2]))
        # the survivors of image 0 are restarts 0, 1 (the ties) and of image 2 restarts 0, 1 (the NaNs): read the map back
        _call(gen, x, R, L, z0, None, [(L - 1, 2)])
        regs = _regions(gen, B, R, [(L - 1, 2)], False)
        assert _read(gen, regs[1], "orig")[:2 * B].tolist()[0:2] == [0, 1]
        assert _read(gen, regs[1], "orig")[:2 * B].tolist()[4:6] == [0, 1]
    finally:
        gen.close()


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_batch_split_and_seeded_z0(precision, weighted):
    arch, B, R, L = "celeba", 6, 3, 9
    w, gen = _gen(arch, precision)
    try:
        x, _, pw = _problem(arch, w, B, R)
        pw = pw if weighted else None
        sched = [(3, 2), (6, 1)]
        whole = _call(gen, x, R, L, None, pw, sched, seed=77)
        drawn = gen.sample_z0(B * R, 77)
        assert _same(_call(gen, x, R, L, drawn, pw, sched), whole)
        for cut in (1, 4):                               # as reconstruct_sharded splits a batch: z_row_offset = first * R
            parts = [_call(gen, x[lo:hi], R, L, None, None if pw is None else pw[lo:hi], sched, seed=77, z_row_offset=lo * R)
                     for lo, hi in ((0, cut), (cut, B))]
            assert _same([torch.cat([p[k] for p in parts]) for k in range(3)], whole), cut
    finally:
        gen.close()


def _regions(gen, batch, R, sched, weighted):
    """{k: {off, n_rows, n_pad, bufs}} of region k of a pruned workspace."""
    return layout(gen, "_pruned", batch, R, list(sched), len(sched), int(weighted))[0]


@pytest.mark.parametrize("precision,arch,weighted", CASES)
def test_gathered_rows_equal_the_source_rows(precision, arch, weighted):
    """A prune point at iter = L - 1: the last stage runs its forward only, so the next region still holds the gathered
    z and v (and z_h), and the first region the state they were gathered from."""
    w, gen = _gen(arch, precision)
    try:
        B, R, L, keep = 5, 4, 8, 2
        x, z0, pw = _problem(arch, w, B, R)
        pw = pw if weighted else None
        sched = [(L - 1, keep)]
        got = _call(gen, x, R, L, z0, pw, sched)
        regs = _regions(gen, B, R, sched, weighted)
        r0, r1 = regs[0], regs[1]
        assert (r0["n_rows"], r1["n_rows"]) == (B * R, B * keep)
        src = _read(gen, r1, "src")[:B * keep].long()
        orig = _read(gen, r1, "orig")[:B * keep].long()
        assert torch.equal(orig, src % R) and torch.equal(src // R, torch.arange(B, device="cuda").repeat_interleave(keep))
        names = ["z", "v"] + (["z_h"] if precision == "fp16" else [])
        for name in names:
            a, b = _read(gen, r0, name), _read(gen, r1, name)
            assert torch.equal(b[:B * keep], a[src]), name
            assert not b[B * keep:].any(), name               # tile-padding rows zeroed
        # the map is the ranking of the loss at iteration L - 2
        want = _composed(gen, x, R, L, z0, pw, sched)
        assert _same(got, want)
        assert torch.equal(got[2].long(), orig.view(B, keep).gather(1, _read(gen, r1, "sel")[:B].long().view(B, 1)).view(B))
    finally:
        gen.close()


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_launch_and_enqueue_counts_and_steady_state(precision, weighted):
    arch, B, R, L = "mnist", 4, 5, 14
    w, gen = _gen(arch, precision)
    try:
        x, z0, pw = _problem(arch, w, B, R)
        pw = pw if weighted else None
        _call(gen, x, R, L, z0, pw, None)
        plain_l, plain_e = gen.last_launch_count, gen.last_enqueue_count
        for sched in (ONE, THREE):
            P = len(sched)
            first = _call(gen, x, R, L, z0, pw, sched)
            assert gen.last_launch_count == plain_l + 3 * P + 1
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            for _ in range(2):                            # replays the captured loop: one graph launch
                assert _same(_call(gen, x, R, L, z0, pw, sched), first)
                assert gen.last_launch_count == plain_l + 3 * P + 1
                assert gen.last_enqueue_count == plain_e + P * (2 if weighted else 1) + 1
            torch.cuda.synchronize()
            assert torch.cuda.mem_get_info()[0] == free0
        assert plain_e + 3 * 2 + 1 <= 14                   # not L-step launches
        # plain calls keep their own graphs and bits next to pruned ones
        again = _call(gen, x, R, L, z0, pw, None)
        assert gen.last_launch_count == plain_l and gen.last_enqueue_count == plain_e
        _, fresh = _gen(arch, precision)
        try:
            assert _same(again, _call(fresh, x, R, L, z0, pw, None))
        finally:
            fresh.close()
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_refused_calls_enqueue_nothing(precision):
    from defensegan_b200 import _native
    arch, B, R, L = "mnist", 3, 4, 10
    w, gen = _gen(arch, precision)
    _, bn = _gen(arch, precision, use_bn=True)
    try:
        lib = gen.lib
        x, z0, _ = _problem(arch, w, B, R)
        hwc = 784
        buf = torch.full((B * hwc + 8,), float("nan"), device="cuda")
        rec = buf[:B * hwc]
        loss = torch.full((B,), float("nan"), device="cuda")

        def sched_of(points):
            return (_native.dgan_prune_point * max(1, len(points)))(*[_native.dgan_prune_point(a, b) for a, b in points])

        good = sched_of([(4, 2)])
        need = int(lib.dgan_workspace_bytes_pruned(gen._handle, B, R, good, 1, 0))
        assert need > 0
        assert int(lib.dgan_workspace_bytes_pruned(bn._handle, B, R, good, 1, 0)) == 0
        assert int(lib.dgan_workspace_bytes_pruned(gen._handle, B, R, sched_of([(4, 5)]), 1, 0)) == 0
        ws_t = torch.empty(need + 1024, dtype=torch.uint8, device="cuda")
        ws = ctypes.c_void_p(ws_base(ws_t))
        prm = _native.dgan_rec_params(B, R, L, 10.0, 0.7, 0, 1, 0)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731

        def call(h, sched, n, x_ptr=p(x), rec_ptr=p(rec), ws_bytes=need):
            return lib.dgan_reconstruct_pruned(h, ctypes.byref(prm), sched, n, x_ptr, None, p(z0), rec_ptr, p(loss), None,
                                               ws, ws_bytes, stream)

        gen.reconstruct(x, R, L, 10.0, z_init_val=z0, prune=[(4, 2)])      # plans, and sets the counts to compare
        launches = gen.last_launch_count
        cases = [
            (gen._handle, sched_of([(L, 2)]), 1, {}, -1, "rec_iters - 1"),
            (gen._handle, sched_of([(4, 2), (4, 1)]), 2, {}, -1, "point 1"),
            (gen._handle, sched_of([(4, 2), (6, 3)]), 2, {}, -1, "point 1"),
            (gen._handle, sched_of([(4, 5)]), 1, {}, -1, "rec_rr"),
            (gen._handle, good, 0, {}, -1, "at least one"),
            (gen._handle, None, 1, {}, -1, "at least one"),
            (gen._handle, good, 1, {"x_ptr": None}, -1, "NULL"),
            (gen._handle, good, 1, {"rec_ptr": ctypes.c_void_p(buf.data_ptr() + 4)}, -1, "16-byte aligned"),
            (bn._handle, good, 1, {}, -3, "use_bn"),
            (gen._handle, good, 1, {"ws_bytes": need - 1}, -4, "dgan_workspace_bytes_pruned"),
        ]
        for h, sched, n, kw, code, msg in cases:
            rc = call(h, sched, n, **kw)
            assert rc == code, (msg, rc)
            assert msg.encode() in lib.dgan_last_error(), (msg, lib.dgan_last_error())
            assert gen.last_launch_count == launches, msg
            torch.cuda.synchronize()
            assert bool(buf.isnan().all()) and bool(loss.isnan().all()), msg
        assert call(gen._handle, good, 1) == 0
        torch.cuda.synchronize()
        assert not bool(rec.isnan().any())
    finally:
        gen.close()
        bn.close()


def test_defensegan_reconstruct_with_rec_prune():
    """DefenseGANBase.reconstruct reads rec_prune at call time and runs the native pruned call; None runs today's call."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp16")
    try:
        gan.rec_rr, gan.rec_iters = 4, 10
        x = torch.tensor(O.synthetic_images("mnist", gan.weights, 3)).cuda()
        z0 = torch.tensor(O.sample_z0(12, 128)).cuda()
        plain = gan.reconstruct(x, z_init_val=z0).clone()
        native = gan._get_native(x.device)
        assert torch.equal(plain, native.reconstruct(x, 4, 10, float(gan.rec_lr), z_init_val=z0))
        gan.rec_prune = [[3, 2], [6, 1]]
        got = gan.reconstruct(x, z_init_val=z0).clone()
        assert torch.equal(got, native.reconstruct(x, 4, 10, float(gan.rec_lr), z_init_val=z0, prune=[(3, 2), (6, 1)]))
        with pytest.raises(ValueError, match="rec_prune"):
            gan.reconstruct_measured(torch.rand(3, 10, device="cuda"), torch.rand(10, 784, device="cuda"))
    finally:
        gan.close()
