"""GPU tests (H100, -m gpu) of the projection from sparse linear measurements (dgan_reconstruct_measured_csr,
dgan_loss_grad_measured_csr) on MNIST and CelebA, with and without BatchNorm:
  - fp32: bit-identical to the dense call on the same matrix (rec, loss and idx at R = 10, L = 200; G, loss and gradient
    of one loop body) for a block average, a 5 x 5 blur, pixel subsampling, a grayscale copy and a random sparse matrix
    with an empty and a fully dense row;
  - fp16: R = 10, L = 200 parity with the measured CPU oracle within test_gpu_measured.py's long-horizon bar;
  - each product against fp64 on the operands it read, read back from the workspace, at 1, 300 and 2560 rows; the staged
    transpose against torch's;
  - steady state: no allocation, the captured loop replayed with the documented counts, and plain, weighted, dense and
    CSR measured calls alternating on one workspace giving the bits of fresh handles' calls;
  - exact homogeneity in the operator's scale;
  - a malformed CSR passed straight to the C-ABI returns NaN, not a fault, and leaves the next call unaffected."""
import ctypes

import numpy as np
import pytest
import torch

import measured_oracle as MO
import sparse_operators as SO
from gpu_support import gen as _gen, layout, release_cached_memory, views  # noqa: F401
from oracle import defensegan_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _release_operators(release_cached_memory):
    """Drop the cached operators before the module's cached memory is handed back."""
    yield
    _OPS.clear()


def _has_guard(gen):
    """The library validates a CSR before using it: its layout names the validity flag."""
    try:
        return "\ncsr_valid i32 " in layout(gen, "_measured_csr", 1, 1, 1)[1]
    except (AttributeError, AssertionError):
        return False


HWC = {"mnist": 784, "celeba": 12288}
SHAPE = {"mnist": (28, 28, 1), "celeba": (64, 64, 3)}
_OPS = {}


def _operator(arch, kind):
    """The dense operator (numpy) of a kind: block2, blur, sub<m>, gray, rand<m>."""
    if (arch, kind) not in _OPS:
        h, w_, c = SHAPE[arch]
        if kind == "block2":
            a = MO.block_average_operator(h, w_, c, 2)
        elif kind == "blur":
            a = SO.blur_operator(h, w_, c)
        elif kind == "gray":
            a = SO.grayscale_operator(h, w_)
        elif kind.startswith("sub"):
            a = SO.subsample_operator(int(kind[3:]), HWC[arch], seed=1)
        else:
            a = SO.random_sparse_operator(int(kind[4:]), HWC[arch], density=0.01, seed=2)
        _OPS[(arch, kind)] = a
    return _OPS[(arch, kind)]


def _lr(a):
    """rec_lr for operator a: reconstruct's step scaled by the share of the image the operator's rows see."""
    m, hwc = a.shape
    return 10.0 * min(1.0, 4.0 * m / hwc) if m < hwc else 10.0


def _problem(arch, kind, w, B, seed=2):
    a = _operator(arch, kind)
    imgs = O.synthetic_images(arch, w, B, kind="S2", seed=seed)
    y = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
    ad = torch.tensor(a).cuda()
    return a, ad, ad.to_sparse_csr(), torch.tensor(y).cuda()


OPS = [("mnist", k) for k in ("block2", "blur", "sub200", "rand100")] + \
      [("celeba", k) for k in ("block2", "blur", "sub2000", "gray", "rand300")]


@pytest.mark.parametrize("use_bn", [False, True])
@pytest.mark.parametrize("arch,kind", OPS)
def test_fp32_csr_is_bit_identical_to_the_dense_call(arch, kind, use_bn):
    w, gen = _gen(arch, "fp32", use_bn)
    try:
        B, R_, L = (3, 10, 200) if arch == "mnist" else (2, 10, 200)
        a, ad, acsr, y = _problem(arch, kind, w, B)
        z0 = torch.tensor(O.sample_z0(B * R_, 128, seed=4)).cuda()
        lr = _lr(a) * (0.05 if use_bn else 1.0)
        dense = gen.reconstruct_measured(y, ad, R_, L, lr, z_init_val=z0, return_aux=True)
        dense = [t.clone() for t in dense]
        sparse = gen.reconstruct_measured(y, acsr, R_, L, lr, z_init_val=z0, return_aux=True)
        assert bool(torch.isfinite(dense[1]).all())
        for name, p, q in zip(("rec", "loss", "idx"), dense, sparse):
            assert torch.equal(p, q), name
        gd = [t.clone() for t in gen.loss_grad_measured(y, ad, z0, R_)]
        gs = gen.loss_grad_measured(y, acsr, z0, R_)
        for name, p, q in zip(("G", "loss", "grad"), gd, gs):
            assert torch.equal(p, q), name
    finally:
        gen.close()


_ORACLE = {}
PARITY = [("mnist", "block2"), ("mnist", "blur"), ("mnist", "sub200"),
          ("celeba", "block2"), ("celeba", "blur"), ("celeba", "sub2000")]


@pytest.mark.parametrize("arch,kind", PARITY)
def test_fp16_long_horizon_parity(arch, kind):
    """R = 10, L = 200 on fp16: per-image |loss_min - oracle| <= 1e-4 (test_long_horizon_measured_parity's bar)."""
    B, R_, L = (4, 10, 200) if arch == "mnist" else (2, 10, 200)
    w, gen = _gen(arch, "fp16")
    try:
        imgs = O.synthetic_images(arch, w, B)
        z0 = O.sample_z0(B * R_, 128)
        a = _operator(arch, kind)
        y = (imgs.reshape(B, -1).astype(np.float64) @ a.T.astype(np.float64)).astype(np.float32)
        if (arch, kind) not in _ORACLE:
            _ORACLE[(arch, kind)] = MO.reconstruct(arch, w, a, y, R_, L, rec_lr=_lr(a), z_init_val=z0)
        ref = _ORACLE[(arch, kind)]
        acsr = torch.tensor(a).cuda().to_sparse_csr()
        rec, loss, idx = gen.reconstruct_measured(torch.tensor(y).cuda(), acsr, R_, L, _lr(a),
                                                  z_init_val=torch.tensor(z0).cuda(), return_aux=True)
        dl = np.abs(loss.cpu().numpy() - ref["loss_min"])
        print("\nfp16 %s %s m=%d: max|dloss|=%.3g (loss %.3g) restart agreement=%.2f"
              % (arch, kind, a.shape[0], dl.max(), float(ref["loss_min"].max()),
                 float((idx.cpu().numpy() == ref["idx"]).mean())))
        assert dl.max() <= 1e-4
    finally:
        gen.close()


def _dense64(rp, ci, v, n_rows, n_cols):
    """The dense fp64 matrix of a staged CSR, and the non-zeros per row."""
    rp = rp.long()
    nnz = int(rp[-1])
    rows = torch.repeat_interleave(torch.arange(n_rows, device=rp.device), rp[1:] - rp[:-1])
    d = torch.zeros(n_rows, n_cols, dtype=torch.float64, device=rp.device)
    d[rows, ci[:nnz].long()] = v[:nnz].double()
    return d, (rp[1:] - rp[:-1]).double()


@pytest.mark.parametrize("n_rows", [1, 300, 2560])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
@pytest.mark.parametrize("arch,kind", [("mnist", "rand100"), ("mnist", "blur"), ("celeba", "block2")])
def test_each_product_on_its_stored_operands(arch, kind, precision, n_rows):
    """r, dy and the loss parts against fp64 on the operands the kernels read: within 1/2 ulp plus (non-zeros in the
    output's row + 1) 2^-24 sum |a||g|; the padded measurements of r and the rows past n_rows exact zeros; the staged
    transpose equal to torch's, order within each row included."""
    w, gen = _gen(arch, precision)
    try:
        u = 2.0 ** -24
        a = _operator(arch, kind)
        m, hwc = a.shape
        acsr = torch.tensor(a).cuda().to_sparse_csr()
        nnz = acsr.values().numel()
        B = max(1, n_rows // 10)
        R_ = n_rows // B
        imgs = torch.tensor(O.synthetic_images(arch, w, B, kind="S2", seed=3)).cuda()
        y = (imgs.reshape(B, -1).double() @ torch.tensor(a).cuda().double().t()).float()
        y += 0.01 * torch.randn(B, m, generator=torch.Generator().manual_seed(1)).cuda()
        z = torch.tensor(O.sample_z0(n_rows, 128, seed=4)).cuda()
        gen.loss_grad_measured(y, acsr, z, R_)           # sizes the workspace
        gen._ws.zero_()
        gen.loss_grad_measured(y, acsr, z, R_)
        torch.cuda.synchronize()
        ws = views(gen, layout(gen, "_measured_csr", n_rows, m, nnz)[0][0])
        assert int(ws["csr_valid"][0]) == 1
        m_ld = ws["r"].shape[1]
        # the staged operator and its transpose
        assert torch.equal(ws["a_rp"][:m + 1].long(), acsr.crow_indices()) and not (ws["a_rp"][m:] - nnz).any()
        assert torch.equal(ws["a_ci"].long(), acsr.col_indices()) and torch.equal(ws["a_v"], acsr.values())
        at = torch.tensor(a).cuda().t().contiguous().to_sparse_csr()
        assert torch.equal(ws["at_rp"].long(), at.crow_indices())
        assert torch.equal(ws["at_ci"].long(), at.col_indices()) and torch.equal(ws["at_v"], at.values())
        A64, k_a = _dense64(ws["a_rp"], ws["a_ci"], ws["a_v"], m_ld, hwc)
        At64, k_at = _dense64(ws["at_rp"], ws["at_ci"], ws["at_v"], hwc, m_ld)
        n = n_rows
        g = ws["y"][:n].double()
        y_rows = ws["ym"][:n // R_].double().repeat_interleave(R_, dim=0)
        r64 = g @ A64.t() - y_rows
        r = ws["r"][:n].double()
        lim = 0.5 * u * r64.abs() + (k_a + 1) * u * (g.abs() @ A64.abs().t() + y_rows.abs()) + 1e-30
        ratio = float(((r - r64).abs() / lim).max())
        assert bool(((r - r64).abs() <= lim).all()), "r: max err / bound %.3g" % ratio
        assert not ws["r"][:n, m:].any() and not ws["r"][n:].any()
        s32 = float(np.float32(2.0) / np.float32(m))
        dy64 = s32 * (r @ At64.t())
        dy = ws["dym"][:n].double()
        lim_dy = 0.5 * u * dy64.abs() + (k_at + 1) * u * s32 * (r.abs() @ At64.abs().t()) + 1e-30
        ratio_dy = float(((dy - dy64).abs() / lim_dy).max())
        assert bool(((dy - dy64).abs() <= lim_dy).all()), "dy: max err / bound %.3g" % ratio_dy
        assert not ws["dym"][n:].any()
        # the loss parts: per 64-column tile, 4-term fmaf chains and a 16-way butterfly over the stored r
        lp = ws["mloss_part"][:, :n].double()
        sq = (r * r).reshape(n, m_ld // 64, 64).sum(dim=2).t()
        assert bool(((lp - sq).abs() <= 8 * u * sq + 1e-30).all())
        assert not ws["mloss_part"][:, n:].any()
        print("\n%s %s %s n=%d: r %.3g, dy %.3g of the bound" % (precision, arch, kind, n_rows, ratio, ratio_dy))
    finally:
        gen.close()


@pytest.mark.parametrize("precision", ["fp16", "fp32"])
def test_steady_state_and_alternating_calls(precision):
    """A second CSR call at a planned size allocates nothing and replays its captured loop with the header's counts; plain,
    weighted, dense and CSR measured calls alternating on one workspace give the bits of fresh handles' calls, and two
    identical calls the same bits."""
    arch, B, R_, L = "mnist", 5, 3, 7
    w, gen = _gen(arch, precision)
    fresh = []
    try:
        a, ad, acsr, y = _problem(arch, "blur", w, B)
        x = torch.tensor(O.synthetic_images(arch, w, B)).cuda()
        z0 = torch.tensor(O.sample_z0(B * R_, 128)).cuda()
        pw = torch.rand(x.shape, generator=torch.Generator().manual_seed(3)).cuda()

        def call(g, kind):
            if kind in ("dense", "csr"):
                out = g.reconstruct_measured(y, ad if kind == "dense" else acsr, R_, L, 1.0, z_init_val=z0, return_aux=True)
            else:
                out = g.reconstruct(x, R_, L, 1.0, z_init_val=z0, return_aux=True,
                                    pixel_weights=pw if kind == "weighted" else None)
            return [t.clone() for t in out]

        want = {}
        for kind in ("csr", "dense", "plain", "weighted"):
            _, g = _gen(arch, precision)
            fresh.append(g)
            want[kind] = call(g, kind)
        for kind in ("csr", "plain", "csr", "dense", "csr", "weighted", "csr", "csr"):
            got = call(gen, kind)
            assert all(torch.equal(p, q) for p, q in zip(got, want[kind])), kind
        call(gen, "plain")
        plain_enq, plain_launches = gen.last_enqueue_count, gen.last_launch_count
        call(gen, "csr")
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        per_step = 6 if precision == "fp16" else 3
        for _ in range(3):
            call(gen, "csr")
            assert gen.last_enqueue_count == plain_enq + 4
            assert gen.last_launch_count == plain_launches + 5 + per_step * (L - 1) + 1
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] == free0
    finally:
        gen.close()
        for g in fresh:
            g.close()


@pytest.mark.parametrize("use_bn", [False, True])
@pytest.mark.parametrize("arch", ["mnist", "celeba"])
@pytest.mark.parametrize("precision", ["fp32", "fp16"])
def test_homogeneity_in_the_operator_scale(precision, arch, use_bn):
    """A and y times 2^k: G bit for bit, the loss and the gradient exactly 4^k times."""
    w, gen = _gen(arch, precision, use_bn)
    try:
        B, R_ = (4, 2) if arch == "mnist" else (2, 2)
        a, ad, acsr, y = _problem(arch, "block2", w, B)
        z = torch.tensor(O.sample_z0(B * R_, 128, seed=6)).cuda()
        g0, l0, d0 = [t.clone() for t in gen.loss_grad_measured(y, acsr, z, R_)]
        for k in (-3, 5):
            s = 2.0 ** k
            g1, l1, d1 = gen.loss_grad_measured(y * s, (ad * s).to_sparse_csr(), z, R_)
            assert torch.equal(g1, g0) and torch.equal(l1, l0 * s * s) and torch.equal(d1, d0 * s * s), k
    finally:
        gen.close()


def test_malformed_csr_through_the_c_abi_gives_nan_and_leaves_the_next_call_alone():
    from defensegan_b200 import _native
    arch, B, R_, L = "mnist", 2, 2, 4
    w, gen = _gen(arch, "fp32")
    try:
        assert _has_guard(gen), "rebuild the library: it does not validate CSR operators"
        a, ad, acsr, y = _problem(arch, "rand100", w, B)
        m, nnz = a.shape[0], acsr.values().numel()
        rp, ci = acsr.crow_indices().int(), acsr.col_indices().int()
        val = acsr.values().contiguous()
        z0 = torch.tensor(O.sample_z0(B * R_, 128)).cuda()
        good = [t.clone() for t in gen.reconstruct_measured(y, acsr, R_, L, 1.0, z_init_val=z0, return_aux=True)]
        ci_bad = ci.clone()
        ci_bad[nnz // 2] = 784 + 1000
        rp_bad = rp.clone()
        rp_bad[3], rp_bad[4] = rp[4], rp[3] - 1          # a decreasing row_ptr (rows 2 and 3 are not empty)
        assert int(rp_bad[4]) < int(rp_bad[3])
        for bad_rp, bad_ci in ((rp, ci_bad), (rp_bad, ci)):
            rec = torch.empty(B, 28, 28, 1, device="cuda")
            loss = torch.empty(B, device="cuda")
            idx = torch.empty(B, dtype=torch.int32, device="cuda")
            ws, need = gen._workspace(B, R_, m=m, nnz=nnz)
            prm = _native.dgan_rec_params(B, R_, L, 1.0, 0.7, 0, 0, 0)
            stream = torch.cuda.current_stream().cuda_stream
            rc = gen.lib.dgan_reconstruct_measured_csr(gen._handle, ctypes.byref(prm), _native._ptr(bad_rp),
                                                       _native._ptr(bad_ci), _native._ptr(val), m, nnz, _native._ptr(y),
                                                       _native._ptr(z0), _native._ptr(rec), _native._ptr(loss),
                                                       _native._ptr(idx), ws, need, ctypes.c_void_p(stream))
            assert rc == 0
            torch.cuda.synchronize()
            assert bool(torch.isnan(loss).all())
            ws_ = views(gen, layout(gen, "_measured_csr", B * R_, m, nnz)[0][0])
            assert int(ws_["csr_valid"][0]) == 0 and not ws_["a_rp"].any() and not ws_["at_rp"].any()
            again = gen.reconstruct_measured(y, acsr, R_, L, 1.0, z_init_val=z0, return_aux=True)
            assert all(torch.equal(p, q) for p, q in zip(again, good))
    finally:
        gen.close()


def test_defensegan_reconstruct_measured_takes_coo_and_csr():
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, precision="fp32")
    gan.rec_rr, gan.rec_iters = 2, 5
    try:
        x = torch.tensor(O.synthetic_images("mnist", O.init_generator_weights("mnist"), 3)).cuda()
        z0 = torch.randn(6, 128, device="cuda") * 128 ** -0.5
        a = torch.tensor(SO.blur_operator(28, 28, 1)).cuda()
        y = x.reshape(3, -1) @ a.t()
        want = gan.reconstruct_measured(y, a, z_init_val=z0)
        for op in (a.to_sparse_csr(), a.to_sparse(), a.cpu().to_sparse()):
            assert torch.equal(gan.reconstruct_measured(y, op, z_init_val=z0), want)
        bad = torch.sparse_csr_tensor(torch.tensor([0, 1]), torch.tensor([784]), torch.ones(1), size=(1, 784),
                                      check_invariants=False)
        with pytest.raises(ValueError, match="column indices"):
            gan.reconstruct_measured(y[:, :1], bad)
    finally:
        gan._drop_native()
