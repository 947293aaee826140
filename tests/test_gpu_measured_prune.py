"""GPU tests (H100, -m gpu) of restart pruning in the projection from linear measurements
(dgan_reconstruct_measured_pruned, dgan_reconstruct_measured_csr_pruned), on MNIST and CelebA, fp32 and fp16, with a
dense Gaussian sketch and sparse operators (tests/sparse_operators.py, the 2x2 block average):
  - an identity schedule (keep = R at every point) gives reconstruct_measured's bits (rec, loss, idx), decay on and off;
  - one- and three-point schedules give the bits of the result composed from rec_rr = 1 measured calls on the tiled
    measurements (rows are independent without BatchNorm);
  - on fp32 the pruned CSR call equals the pruned dense call on the same matrix bit for bit;
  - ties keep the lower original index; an image with a NaN measurement returns restart 0;
  - a malformed CSR gives NaN losses and an idx in [0, R), and leaves the next valid call's bits alone;
  - the layout: the operator block once, then the regions; the gathered z / v (/ z_h) rows equal their source rows;
  - the header's launch and enqueue counts, a replayed graph and no allocation in steady state;
  - measured, pruned measured, plain and pruned plain calls alternating on one handle give fresh handles' bits;
  - the workspace is the operator block plus the regions, well under (P + 1) unpruned measured workspaces;
  - use_bn and the argument checks refuse before anything is enqueued."""
import ctypes

import numpy as np
import pytest
import torch

import measured_oracle as MO
import sparse_operators as SO
from gpu_support import bits as _bits, gen as _gen, layout
from gpu_support import read as _read, release_cached_memory, same as _same, ws_base  # noqa: F401
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu

HWC = {"mnist": 784, "celeba": 12288}
SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}
ONE = [(5, 2)]
THREE = [(3, 3), (6, 2), (9, 1)]
# (operator kind, passed as CSR): a dense Gaussian sketch, the 2x2 block average and pixel subsampling as CSR
OPS = [("gauss", False), ("block2", True), ("sub", True)]
CASES = [(p, a, k, c) for p in ("fp32", "fp16") for a in ("mnist", "celeba") for k, c in OPS]


def _operator(arch, kind):
    h, w_, c = SHAPE[arch]
    if kind == "block2":
        return MO.block_average_operator(h, w_, c, 2)
    if kind == "sub":
        return SO.subsample_operator(HWC[arch] // 6, HWC[arch], seed=1)
    return MO.gaussian_operator(100 if arch == "mnist" else 500, HWC[arch], seed=5)


def _problem(arch, kind, csr, w, B, R, seed=2):
    """(operator as passed, y [B, m], z0 [B*R, 128], rec_lr)."""
    a = _operator(arch, kind)
    imgs = O.synthetic_images(arch, w, B, kind="S2", seed=seed)
    y = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
    ad = torch.tensor(a).cuda()
    z0 = torch.tensor(O.sample_z0(B * R, 128, seed=seed + 1)).cuda()
    lr = 10.0 * min(1.0, 4.0 * a.shape[0] / a.shape[1])
    return (ad.to_sparse_csr() if csr else ad), torch.tensor(y).cuda(), z0, lr


def _call(gen, y, op, R, L, z0, lr, prune, decay=False, **kw):
    return [t.clone() for t in gen.reconstruct_measured(y, op, R, L, lr, z_init_val=z0, prune=prune, decay_lr=decay,
                                                        return_aux=True, **kw)]


def _before(a, b):
    """prune_before of kernels_prune.cuh on (loss, original index) pairs."""
    (la, oa), (lb, ob) = a, b
    na, nb = np.isnan(la), np.isnan(lb)
    if na or nb:
        return (nb and oa < ob) if na else True
    return la < lb or (la == lb and oa < ob)


def _composed(gen, y, op, R, L, z0, lr, prune):
    """The pruned call's result from rec_rr = 1 measured calls on the tiled measurements (decay_lr off)."""
    B = y.shape[0]
    yt = y.repeat_interleave(R, dim=0)
    loss_at = {it: _call(gen, yt, op, 1, it, z0, lr, None)[1].cpu().numpy() for it, _ in prune}
    rec_all, loss_all, _ = _call(gen, yt, op, 1, L, z0, lr, None)
    loss_all = loss_all.cpu().numpy()
    rec = torch.empty((B,) + tuple(rec_all.shape[1:]), device="cuda")
    loss, idx = torch.empty(B, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda")
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
@pytest.mark.parametrize("precision,arch,kind,csr", CASES)
def test_identity_schedule_gives_the_measured_bits(precision, arch, kind, csr, decay):
    w, gen = _gen(arch, precision)
    try:
        B, R, L = 3, 4, 12
        op, y, z0, lr = _problem(arch, kind, csr, w, B, R)
        plain = _call(gen, y, op, R, L, z0, lr, None, decay=decay)
        assert bool(torch.isfinite(plain[1]).all())
        for sched in ([(5, R)], [(1, R), (6, R), (11, R)]):
            assert _same(_call(gen, y, op, R, L, z0, lr, sched, decay=decay), plain), sched
    finally:
        gen.close()


@pytest.mark.parametrize("sched", [ONE, THREE], ids=["one", "three"])
@pytest.mark.parametrize("precision,arch,kind,csr", CASES)
def test_pruned_call_equals_the_composed_result(precision, arch, kind, csr, sched):
    w, gen = _gen(arch, precision)
    try:
        B, R, L = 5, 4, 12
        op, y, z0, lr = _problem(arch, kind, csr, w, B, R)
        got = _call(gen, y, op, R, L, z0, lr, sched)
        assert _same(got, _composed(gen, y, op, R, L, z0, lr, sched))
        assert int(got[2].min()) >= 0 and int(got[2].max()) < R
    finally:
        gen.close()


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_fp32_pruned_csr_equals_the_pruned_dense_call(arch):
    w, gen = _gen(arch, "fp32")
    try:
        B, R, L = 4, 5, 12
        for kind in ("block2", "gauss"):
            ad, y, z0, lr = _problem(arch, kind, False, w, B, R)
            for sched in (ONE, THREE):
                dense = _call(gen, y, ad, R, L, z0, lr, sched)
                assert _same(_call(gen, y, ad.to_sparse_csr(), R, L, z0, lr, sched), dense), (kind, sched)
    finally:
        gen.close()


@pytest.mark.parametrize("csr", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_ties_keep_the_lower_index_and_nan_images_keep_restart_0(precision, csr):
    arch, B, R, L = "mnist", 3, 4, 10
    w, gen = _gen(arch, precision)
    try:
        op, y, z0, lr = _problem(arch, "block2", csr, w, B, R)
        z0[1:R] = z0[0]                                  # image 0: four identical restarts, identical losses
        y[2, 3] = float("nan")                           # image 2: every loss NaN
        for sched in ([(4, 2)], [(2, 3), (6, 1)]):
            got = _call(gen, y, op, R, L, z0, lr, sched)
            assert _same(got, _composed(gen, y, op, R, L, z0, lr, sched)), sched
            assert int(got[2][0]) == 0 and int(got[2][2]) == 0, sched
            assert bool(torch.isnan(got[1][2])) and not bool(torch.isnan(got[1][:2]).any())
    finally:
        gen.close()


def test_malformed_csr_gives_nan_and_leaves_the_next_call_alone():
    from defensegan_b200 import _native
    arch, B, R, L = "mnist", 3, 4, 8
    w, gen = _gen(arch, "fp32")
    try:
        acsr, y, z0, lr = _problem(arch, "block2", True, w, B, R)
        m, nnz = acsr.shape[0], acsr.values().numel()
        rp, ci, val = acsr.crow_indices().int(), acsr.col_indices().int(), acsr.values().contiguous()
        sched = [(3, 2), (6, 1)]
        good = _call(gen, y, acsr, R, L, z0, lr, sched)
        ci_bad = ci.clone()
        ci_bad[nnz // 2] = 784 + 1000
        arr = (_native.dgan_prune_point * 2)(*[_native.dgan_prune_point(a, b) for a, b in sched])
        rec = torch.empty(B, 28, 28, 1, device="cuda")
        loss = torch.empty(B, device="cuda")
        idx = torch.full((B,), -7, dtype=torch.int32, device="cuda")
        ws, need = gen._workspace(B, R, m=m, nnz=nnz, sched=arr)
        prm = _native.dgan_rec_params(B, R, L, lr, 0.7, 0, 0, 0)
        stream = torch.cuda.current_stream().cuda_stream
        rc = gen.lib.dgan_reconstruct_measured_csr_pruned(gen._handle, ctypes.byref(prm), arr, 2, _native._ptr(rp),
                                                          _native._ptr(ci_bad), _native._ptr(val), m, nnz, _native._ptr(y),
                                                          _native._ptr(z0), _native._ptr(rec), _native._ptr(loss),
                                                          _native._ptr(idx), ws, need, ctypes.c_void_p(stream))
        assert rc == 0
        torch.cuda.synchronize()
        assert bool(torch.isnan(loss).all())
        assert int(idx.min()) >= 0 and int(idx.max()) < R
        assert idx.tolist() == [0] * B                   # every loss NaN: survivors 0 .. keep - 1, then restart 0
        assert _same(_call(gen, y, acsr, R, L, z0, lr, sched), good)
    finally:
        gen.close()


# ---- the workspace ----

def _layout(gen, batch, R, m, nnz, sched):
    """{"operator": the operator block, k: region k}, each {off, n_rows, n_pad, bufs}, in that order."""
    return layout(gen, "_measured_pruned", batch, R, m, nnz, list(sched), len(sched))[0]


def _block_bytes(block):
    size = {"f32": 4, "f16": 2, "u64": 8, "u32": 4, "i32": 4}
    return max(off + (int(np.prod(d)) * size[t] + 1023) // 1024 * 1024 for t, off, d in block["bufs"].values())


@pytest.mark.parametrize("csr", [False, True])
def test_layout_is_the_operator_block_once_then_the_regions(csr):
    from defensegan_b200 import _native
    w, gen = _gen("celeba", "fp16")
    try:
        B, R, m = 8, 10, 2000
        nnz = 30000 if csr else -1
        for sched in (ONE, THREE, [(40, 2)], [(20, 5), (60, 2), (120, 1)]):
            regions = _layout(gen, B, R, m, nnz, sched)
            assert list(regions) == ["operator"] + list(range(len(sched) + 1))
            blocks = list(regions.values())
            op = blocks[0]
            m_ld = (m + 63) // 64 * 64
            if csr:
                assert "am" not in op["bufs"] and op["bufs"]["a_ci"][2] == [nnz]
                assert op["bufs"]["at_rp"][2] == [12288 + 1]
            else:
                assert op["bufs"]["am"][2] == [m_ld, 12288] and op["bufs"]["amt"][2] == [12288, m_ld]
            assert op["bufs"]["ym"][2] == [B, m_ld] and op["off"] == 0 and op["n_rows"] == B
            off = _block_bytes(op)
            for k, reg in enumerate(blocks[1:]):
                assert reg["off"] == off, k
                assert reg["n_rows"] == B * (R if k == 0 else sched[k - 1][1])
                names = set(reg["bufs"])
                assert {"z", "v", "y", "r", "dym", "mloss_part", "mscale", "orig", "src", "sel"} <= names
                assert not names & {"am", "amt", "ym", "a_rp", "a_ci", "a_v", "at_rp", "at_ci", "at_v", "csr_bad",
                                    "csr_valid"}
                assert reg["bufs"]["r"][2] == [reg["n_pad"], m_ld]
                off += _block_bytes(reg)
            arr = (_native.dgan_prune_point * len(sched))(*[_native.dgan_prune_point(a, b) for a, b in sched])
            pruned = int(gen.lib.dgan_workspace_bytes_measured_pruned(gen._handle, B, R, m, nnz, arr, len(sched)))
            assert pruned == off, sched
        # dense CelebA at m = 2000: the operator is staged once, not once per stage
        B, R = 128, 10
        for sched in ([(40, 2)], [(20, 5), (60, 2), (120, 1)]):
            arr = (_native.dgan_prune_point * len(sched))(*[_native.dgan_prune_point(a, b) for a, b in sched])
            pruned = int(gen.lib.dgan_workspace_bytes_measured_pruned(gen._handle, B, R, m, -1, arr, len(sched)))
            unpruned = int(gen.lib.dgan_workspace_bytes_measured(gen._handle, B, R, m))
            print("\nCelebA B=%d R=%d m=%d %s: pruned measured workspace %.1f MB, unpruned %.1f MB"
                  % (B, R, m, sched, pruned / 2 ** 20, unpruned / 2 ** 20))
            assert 0 < pruned < (len(sched) + 1) * unpruned
    finally:
        gen.close()


@pytest.mark.parametrize("precision,arch,kind,csr", [c for c in CASES if c[2] != "sub"])
def test_gathered_rows_equal_the_source_rows(precision, arch, kind, csr):
    """A prune point at iter = L - 1: the last stage runs its forward only, so the next region still holds the gathered
    z and v (and z_h), and the first region the state they were gathered from."""
    w, gen = _gen(arch, precision)
    try:
        B, R, L, keep = 5, 4, 8, 2
        op, y, z0, lr = _problem(arch, kind, csr, w, B, R)
        sched = [(L - 1, keep)]
        got = _call(gen, y, op, R, L, z0, lr, sched)
        nnz = op.values().numel() if csr else -1
        blocks = list(_layout(gen, B, R, op.shape[0], nnz, sched).values())
        r0, r1 = blocks[1], blocks[2]
        assert (r0["n_rows"], r1["n_rows"]) == (B * R, B * keep)
        src = _read(gen, r1, "src")[:B * keep].long()
        orig = _read(gen, r1, "orig")[:B * keep].long()
        assert torch.equal(orig, src % R) and torch.equal(src // R, torch.arange(B, device="cuda").repeat_interleave(keep))
        for name in ["z", "v"] + (["z_h"] if precision == "fp16" else []):
            a, b = _read(gen, r0, name), _read(gen, r1, name)
            assert torch.equal(b[:B * keep], a[src]), name
            assert not b[B * keep:].any(), name           # tile-padding rows zeroed
        assert torch.equal(got[2].long(), orig.view(B, keep).gather(1, _read(gen, r1, "sel")[:B].long().view(B, 1)).view(B))
        # the operator block holds the staged measurements once, for the batch's images
        ym = _read(gen, blocks[0], "ym")
        assert torch.equal(ym[:, :y.shape[1]], y) and not ym[:, y.shape[1]:].any()
        # the map is the ranking of the measured loss at iteration L - 2 (the composed calls reuse the workspace)
        assert _same(got, _composed(gen, y, op, R, L, z0, lr, sched))
    finally:
        gen.close()


@pytest.mark.parametrize("csr", [False, True])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_launch_and_enqueue_counts_and_steady_state(precision, csr):
    arch, B, R, L = "mnist", 4, 5, 14
    w, gen = _gen(arch, precision)
    try:
        op, y, z0, lr = _problem(arch, "block2", csr, w, B, R)
        _call(gen, y, op, R, L, z0, lr, None)
        meas_l, meas_e = gen.last_launch_count, gen.last_enqueue_count
        for sched in (ONE, THREE):
            P = len(sched)
            first = _call(gen, y, op, R, L, z0, lr, sched)
            assert gen.last_launch_count == meas_l + 3 * P + 1
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            for _ in range(2):                            # replays the captured loop: one graph launch
                assert _same(_call(gen, y, op, R, L, z0, lr, sched), first)
                assert gen.last_launch_count == meas_l + 3 * P + 1
                assert gen.last_enqueue_count == meas_e + 1
            torch.cuda.synchronize()
            assert torch.cuda.mem_get_info()[0] == free0
        again = _call(gen, y, op, R, L, z0, lr, None)
        assert gen.last_launch_count == meas_l and gen.last_enqueue_count == meas_e
        _, fresh = _gen(arch, precision)
        try:
            assert _same(again, _call(fresh, y, op, R, L, z0, lr, None))
        finally:
            fresh.close()
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_alternating_kinds_on_one_handle_give_fresh_handles_bits(precision):
    """Measured, pruned measured (dense and CSR), plain and pruned plain calls on one handle and workspace: no two kinds
    share a captured graph."""
    arch, B, R, L = "mnist", 4, 4, 10
    w, gen = _gen(arch, precision)
    fresh = []
    try:
        ad, y, z0, lr = _problem(arch, "block2", False, w, B, R)
        acsr = ad.to_sparse_csr()
        x = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=2)).cuda()
        sched = [(3, 2), (6, 1)]

        def call(g, kind):
            if kind == "plain":
                out = g.reconstruct(x, R, L, lr, z_init_val=z0, return_aux=True)
            elif kind == "plain-pruned":
                out = g.reconstruct(x, R, L, lr, z_init_val=z0, return_aux=True, prune=sched)
            else:
                op = acsr if kind.startswith("csr") else ad
                out = g.reconstruct_measured(y, op, R, L, lr, z_init_val=z0, return_aux=True,
                                             prune=sched if kind.endswith("pruned") else None)
            return [t.clone() for t in out]

        kinds = ("dense", "dense-pruned", "csr", "csr-pruned", "plain", "plain-pruned")
        want = {}
        for kind in kinds:
            _, g = _gen(arch, precision)
            fresh.append(g)
            want[kind] = call(g, kind)
        for kind in ("dense-pruned", "plain", "csr-pruned", "dense", "plain-pruned", "dense-pruned", "csr", "csr-pruned",
                     "plain", "dense-pruned"):
            assert _same(call(gen, kind), want[kind]), kind
    finally:
        gen.close()
        for g in fresh:
            g.close()


@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_refused_calls_enqueue_nothing(precision):
    from defensegan_b200 import _native
    arch, B, R, L = "mnist", 3, 4, 10
    w, gen = _gen(arch, precision)
    _, bn = _gen(arch, precision, use_bn=True)
    try:
        lib = gen.lib
        ad, y, z0, lr = _problem(arch, "block2", False, w, B, R)
        acsr = ad.to_sparse_csr()
        m = ad.shape[0]
        rp, ci, val = acsr.crow_indices().int(), acsr.col_indices().int(), acsr.values().contiguous()
        nnz = val.numel()
        buf = torch.full((B * 784 + 8,), float("nan"), device="cuda")
        rec = buf[:B * 784]
        loss = torch.full((B,), float("nan"), device="cuda")

        def sched_of(points):
            return (_native.dgan_prune_point * max(1, len(points)))(*[_native.dgan_prune_point(a, b) for a, b in points])

        good = sched_of([(4, 2)])
        need = int(lib.dgan_workspace_bytes_measured_pruned(gen._handle, B, R, m, nnz, good, 1))
        assert need > 0
        assert int(lib.dgan_workspace_bytes_measured_pruned(bn._handle, B, R, m, nnz, good, 1)) == 0
        assert int(lib.dgan_workspace_bytes_measured_pruned(gen._handle, B, R, m, nnz, sched_of([(4, 5)]), 1)) == 0
        for bad_m, bad_nnz in ((0, -1), (785, -1), (m, -2), (m, m * 784 + 1)):
            assert int(lib.dgan_workspace_bytes_measured_pruned(gen._handle, B, R, bad_m, bad_nnz, good, 1)) == 0
        ws_t = torch.empty(need + 1024, dtype=torch.uint8, device="cuda")
        ws = ctypes.c_void_p(ws_base(ws_t))
        prm = _native.dgan_rec_params(B, R, L, lr, 0.7, 0, 1, 0)
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        p = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731

        def dense(h, sched, n, a_ptr=p(ad), m_=m, rec_ptr=p(rec), ws_bytes=need):
            return lib.dgan_reconstruct_measured_pruned(h, ctypes.byref(prm), sched, n, a_ptr, m_, p(y), p(z0), rec_ptr,
                                                        p(loss), None, ws, ws_bytes, stream)

        def csr(h, sched, n, rp_ptr=p(rp), m_=m, nnz_=nnz, rec_ptr=p(rec), ws_bytes=need):
            return lib.dgan_reconstruct_measured_csr_pruned(h, ctypes.byref(prm), sched, n, rp_ptr, p(ci), p(val), m_, nnz_,
                                                            p(y), p(z0), rec_ptr, p(loss), None, ws, ws_bytes, stream)

        gen.reconstruct_measured(y, acsr, R, L, lr, z_init_val=z0, prune=[(4, 2)])     # plans; the counts to compare
        launches = gen.last_launch_count
        misaligned = ctypes.c_void_p(buf.data_ptr() + 4)
        cases = []
        for fn in (dense, csr):
            cases += [
                (fn, gen._handle, sched_of([(L, 2)]), 1, {}, -1, "rec_iters - 1"),
                (fn, gen._handle, sched_of([(4, 2), (6, 3)]), 2, {}, -1, "point 1"),
                (fn, gen._handle, sched_of([(4, 5)]), 1, {}, -1, "rec_rr"),
                (fn, gen._handle, None, 1, {}, -1, "at least one"),
                (fn, gen._handle, good, 1, {"rec_ptr": misaligned}, -1, "16-byte aligned"),
                (fn, gen._handle, good, 1, {"m_": 785}, -1, "m = 785"),
                (fn, bn._handle, good, 1, {}, -3, "use_bn"),
            ]
        need_dense = int(lib.dgan_workspace_bytes_measured_pruned(gen._handle, B, R, m, -1, good, 1))
        cases += [
            (dense, gen._handle, good, 1, {"a_ptr": None}, -1, "NULL operator"),
            (dense, gen._handle, good, 1, {"ws_bytes": need_dense - 1}, -4, "dgan_workspace_bytes_measured_pruned"),
            (csr, gen._handle, good, 1, {"rp_ptr": None}, -1, "NULL row_ptr"),
            (csr, gen._handle, good, 1, {"nnz_": m * 784 + 1}, -1, "nnz ="),
            (csr, gen._handle, good, 1, {"ws_bytes": need - 1}, -4, "dgan_workspace_bytes_measured_pruned"),
        ]
        for fn, h, sched, n, kw, code, msg in cases:
            rc = fn(h, sched, n, **kw)
            assert rc == code, (fn.__name__, msg, rc)
            assert msg.encode() in lib.dgan_last_error(), (msg, lib.dgan_last_error())
            assert gen.last_launch_count == launches, msg
            torch.cuda.synchronize()
            assert bool(buf.isnan().all()) and bool(loss.isnan().all()), msg
        assert csr(gen._handle, good, 1) == 0
        torch.cuda.synchronize()
        assert not bool(rec.isnan().any())
    finally:
        gen.close()
        bn.close()


def test_defensegan_reconstruct_measured_with_prune():
    """DefenseGANBase.reconstruct_measured(prune=...) runs the native pruned call for dense, COO and CSR operators;
    prune=None runs today's call whatever rec_prune holds, and without prune a set rec_prune is still refused."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp16")
    try:
        gan.rec_rr, gan.rec_iters = 4, 10
        a = torch.tensor(MO.block_average_operator(28, 28, 1, 2)).cuda()
        x = torch.tensor(O.synthetic_images("mnist", gan.weights, 3)).cuda()
        y = x.reshape(3, -1) @ a.t()
        z0 = torch.tensor(O.sample_z0(12, 128)).cuda()
        native = gan._get_native(a.device)
        sched = [(3, 2), (6, 1)]
        for op in (a, a.to_sparse(), a.to_sparse_csr()):
            want = native.reconstruct_measured(y, op.to_sparse_csr() if op.layout == torch.sparse_coo else op, 4, 10,
                                               float(gan.rec_lr), z_init_val=z0, prune=sched).clone()
            assert torch.equal(gan.reconstruct_measured(y, op, z_init_val=z0, prune=[[3, 2], [6, 1]]), want)
        plain = gan.reconstruct_measured(y, a, z_init_val=z0).clone()
        gan.rec_prune = [(2, 1)]
        assert torch.equal(gan.reconstruct_measured(y, a, z_init_val=z0, prune=None), plain)
        with pytest.raises(ValueError, match="rec_prune"):
            gan.reconstruct_measured(y, a, z_init_val=z0)
    finally:
        gan.close()
