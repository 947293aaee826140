"""CPU tests of the host side: C-ABI library loads and exports every declared symbol, the
reference-mirroring Python surface, config/flags, the eval driver and the shard/gather logic
(gloo, world_size 2)."""
import argparse
import os
import re
import socket
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_header_symbol():
    from defensegan_b200 import _native
    _native.build_library()
    lib = _native.load_library()
    header = open(os.path.join(ROOT, "include", "defensegan_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(dgan_[a-z0-9_]+)\s*\(", header)))
    assert declared, "no declarations parsed"
    for sym in declared:
        assert hasattr(lib, sym), "library does not export %s" % sym
    assert sorted(declared) == sorted(_native.ABI_SYMBOLS)
    assert lib.dgan_abi_version() == 2
    d = _native.dgan_desc(_native.ABI_VERSION, 0, 128, 64, 0, 0)
    import ctypes
    assert lib.dgan_num_weights(ctypes.byref(d)) == 8
    d.arch = 1
    assert lib.dgan_num_weights(ctypes.byref(d)) == 10


def test_no_cpu_fallback():
    if torch.cuda.is_available():
        pytest.skip("CUDA present")
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    with pytest.raises(RuntimeError):
        gan.reconstruct(torch.zeros(2, 28, 28, 1))


def test_model_classes_mirror_reference_defaults(tmp_path):
    from defensegan_b200.models import gan as G
    m = G.MnistDefenseGAN(test_mode=True, verbose=False)
    assert (m.rec_iters, m.rec_rr, m.rec_lr) == (200, 10, 10.0)
    assert (m.latent_dim, m.net_dim, m.use_bn, m.batch_size) == (128, 64, False, 50)
    assert m.image_dim == [28, 28, 1] and m.dataset_name == "mnist" and m.test_batch_size == m.batch_size
    assert m.checkpoint_dir == os.path.join("output", "gans", "mnist")
    f = G.FmnistDefenseDefenseGAN(test_mode=True, verbose=False)
    assert f.dataset_name == "f-mnist" and f.arch == "mnist"
    c = G.CelebADefenseGAN(test_mode=True, verbose=False)
    assert c.rec_rr == 2 and c.image_dim == [64, 64, 3]
    assert set(G.dataset_gan_dict) == {"mnist", "f-mnist", "celeba"}
    # callers override hyper-parameters after construction (blackbox.py:649-658)
    m.rec_rr, m.rec_lr, m.rec_iters = 2, 1.0, 10
    # batch_size % rec_rr assertion (models/gan.py:101-104)
    with pytest.raises(AssertionError):
        G.MnistDefenseGAN(test_mode=True, verbose=False, batch_size=32, rec_rr=10)
    with pytest.raises(TypeError):
        G.MnistDefenseGAN(test_mode=True, verbose=False, not_an_attribute=1)
    # input transforms (models/gan.py:684-685,764-765)
    assert float(m.input_transform(np.array([255.0]))[0]) == 1.0
    assert float(c.input_transform(np.array([0.0]))[0]) == -1.0
    # checkpoint round trip
    p = m.save_generator(str(tmp_path))
    m2 = G.MnistDefenseGAN(test_mode=True, verbose=False, seed=7)
    assert not np.array_equal(m2.weights["Generator.Input/Generator.Input.W"], m.weights["Generator.Input/Generator.Input.W"])
    assert m2.load_generator(str(tmp_path)) is True and os.path.isfile(p)
    np.testing.assert_array_equal(m2.weights["Generator.3/Generator.3.Filters"], m.weights["Generator.3/Generator.3.Filters"])
    assert m2.load_generator(str(tmp_path / "missing")) is False


def test_weight_init_matches_oracle():
    from defensegan_b200 import weights as W
    from oracle import defensegan_oracle as O
    for arch in ("mnist", "celeba"):
        a, b = W.init_generator_weights(arch), O.init_generator_weights(arch)
        assert list(a.keys()) == list(b.keys())
        for k in a:
            np.testing.assert_array_equal(a[k], b[k])
    with pytest.raises(ValueError):
        W.validate_weights("mnist", {k: v[..., :1] for k, v in a.items()}, 128, 64, False)


def test_config_and_flags():
    from defensegan_b200.utils import config as C
    cfg = C.load_config(C.packaged_cfg_path("mnist"))
    assert cfg["REC_ITERS"] == 200 and cfg["REC_RR"] == 10 and cfg["REC_LR"] == 10.0
    assert cfg["LATENT_DIM"] == 128 and cfg["USE_BN"] is False and cfg["IMAGE_DIM"] == [28, 28, 1]
    parser = C.add_flags(argparse.ArgumentParser(), cfg)
    ns = parser.parse_args(["--rec_iters", "20", "--rec_lr", "1.5", "--rec_rr", "5", "--use_bn", "False"])
    over = C.flags_to_cfg(ns, cfg)
    assert (over["REC_ITERS"], over["REC_LR"], over["REC_RR"], over["USE_BN"]) == (20, 1.5, 5, False)
    from defensegan_b200.models.gan import MnistDefenseGAN
    m = MnistDefenseGAN(cfg=over, test_mode=True, verbose=False)
    assert (m.rec_iters, m.rec_lr, m.rec_rr) == (20, 1.5, 5)
    with pytest.raises(IOError):
        C.load_config("/nonexistent/x.yml")


def test_model_eval_gan_eager_contract():
    from defensegan_b200.utils.gan_defense import model_eval_gan, SharedReconstruction
    n, bs = 10, 4
    x = np.random.RandomState(0).rand(n, 28, 28, 1).astype("f4")
    labels = np.eye(10, dtype="f4")[np.arange(n) % 10]
    calls = []

    class FakeGan:
        def reconstruct(self, xb, **kw):
            calls.append(int(xb.shape[0]))
            return xb * 0.5

    rec = SharedReconstruction(FakeGan())

    def predictions(xb):
        r = rec(xb)
        out = torch.zeros(xb.shape[0], 10)
        out[torch.arange(xb.shape[0]), (torch.arange(xb.shape[0]) + len(seen)) % 10] = 1.0
        seen.extend(range(xb.shape[0]))
        return out

    seen = []
    acc, roc = model_eval_gan(None, None, None, predictions=predictions, test_images=x, test_labels=labels,
                              args={"batch_size": bs}, diff_op=lambda xb: ((xb - rec(xb)) ** 2).mean(dim=(1, 2, 3)),
                              device=torch.device("cpu"))
    assert calls == [4, 4, 2]                      # one projection per batch, ragged tail kept
    assert acc == 1.0 and len(roc[0]) == n and len(roc[1]) == n and roc[2].shape == (n,)
    np.testing.assert_allclose(roc[2], ((x * 0.5) ** 2).mean(axis=(1, 2, 3)), rtol=1e-5)
    with pytest.raises(AssertionError):
        model_eval_gan(None, None, None, predictions=predictions, test_images=x, test_labels=labels, args={})
    with pytest.raises(ValueError):
        model_eval_gan(None, None, None, predictions=predictions, args={"batch_size": 2})
    acc2, acc_rec, roc2 = model_eval_gan(None, None, None, predictions=lambda xb: torch.ones(len(xb), 10),
                                         predictions_rec=lambda xb: torch.ones(len(xb), 10), test_images=x,
                                         test_labels=labels, args={"batch_size": bs}, device=torch.device("cpu"))
    assert abs(acc2 - 0.1) < 1e-9 and abs(acc_rec - 0.1) < 1e-9


def test_shard_bounds():
    from defensegan_b200.parallel import shard_bounds
    assert shard_bounds(4096, 8) == [512 * i for i in range(9)]
    assert shard_bounds(10, 4) == [0, 3, 6, 8, 10]
    assert shard_bounds(2, 4) == [0, 1, 2, 2, 2]


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
        z0 = torch.rand(n_images * rec_rr, 8, generator=g)

        def local_fn(x, z, out, first_image):
            # stand-in for the per-rank projection: depends on the image AND its R z0 rows
            out.copy_(x * 2.0 + z.reshape(x.shape[0], rec_rr, -1).sum(dim=(1, 2)).view(-1, 1, 1, 1))

        got = sharded_apply(local_fn, images, rec_rr, z_init_val=z0)
        want = images * 2.0 + z0.reshape(n_images, rec_rr, -1).sum(dim=(1, 2)).view(-1, 1, 1, 1)
        ok = bool(torch.equal(got, want))

        # z_init_val=None: every shard must index ONE common z0 stream at (first image) * rec_rr - stand-in for the
        # native Philox draw: "z0 row r" = r, so the single-device result is image-independent and known
        def local_rand(x, z, out, first_image):
            assert z is None
            rows = first_image * rec_rr + torch.arange(x.shape[0] * rec_rr, dtype=torch.float32)
            out.copy_(rows.reshape(x.shape[0], rec_rr).sum(dim=1).view(-1, 1, 1, 1).expand_as(x))

        got = sharded_apply(local_rand, images, rec_rr, z_init_val=None)
        want = torch.arange(n_images * rec_rr, dtype=torch.float32).reshape(n_images, rec_rr).sum(dim=1)
        ok = ok and bool(torch.equal(got[:, 0, 0, 0], want))
        ret[rank] = ok
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("n_images", [8, 5])
def test_sharded_gather_gloo_world2(n_images):
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


def test_reconstruct_dataset_cache_format(tmp_path, monkeypatch):
    """f1 (reference models/gan.py:451-587): directory naming, per-image pickles, feats.pkl short-cut and the
    regex the callers use to parse hyper-parameters back out of the path (blackbox.py:646-651)."""
    import pickle
    import re
    from defensegan_b200.models.gan import MnistDefenseGAN
    gan = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=str(tmp_path))
    gan.initialized = True
    gan.rec_rr, gan.rec_lr, gan.rec_iters = 2, 0.5, 3
    calls = []

    def fake_reconstruct(x, **kw):                 # the projector needs a GPU; the cache logic does not
        calls.append(int(x.shape[0]))
        return x * 0.5

    monkeypatch.setattr(gan, "reconstruct", fake_reconstruct)
    rs = np.random.RandomState(0)
    data = {sp: (rs.randint(0, 256, size=(n, 28, 28, 1)).astype("uint8"), np.arange(n) % 10)
            for sp, n in (("train", 5), ("dev", 3), ("test", 4))}

    def gen(sp, bs=2):
        def g():
            x, y = data[sp]
            for i in range(0, len(x), bs):
                yield x[i:i + bs], y[i:i + bs]
        return g

    gan.set_dataset_generators(train=gen("train"), dev=gen("dev"), test=gen("test"))
    rets = gan.reconstruct_dataset()
    assert calls == [2, 2, 1, 2, 1, 2, 2]
    d = gan.rec_cache_dir("test")
    assert d == os.path.join(str(tmp_path), "gans", "mnist", "recs_rr2_lr0.50000_iters3", "test")
    assert re.compile("recs_rr(.*)_lr(.*)_iters(.*)").findall(os.path.dirname(d))[0] == ("2", "0.50000", "3")
    recs, targets, orig = rets["test"]
    assert recs.shape == (4, 28, 28, 1) and orig.shape == (4, 28, 28, 1) and list(targets) == [0, 1, 2, 3]
    np.testing.assert_allclose(orig, data["test"][0] / 255.0, rtol=1e-6)
    np.testing.assert_allclose(recs, orig * 0.5, rtol=1e-6)
    with open(os.path.join(d, "pickles", "rec_0000003_l3.pkl"), "rb") as f:
        np.testing.assert_allclose(pickle.load(f), recs[3])
    # a ragged last batch keeps its position in the split (5 images in batches of 2: the last one is image 4)
    assert os.path.isfile(os.path.join(gan.rec_cache_dir("train"), "pickles", "rec_0000004_l4.pkl"))
    # second call: every batch comes from the per-image cache, no projection runs
    calls.clear()
    rets2 = gan.reconstruct_dataset()
    assert calls == []
    np.testing.assert_array_equal(rets2["train"][0], rets["train"][0])
    # feats.pkl short-cut
    gan.save_recs(rets)
    assert os.path.isfile(os.path.join(d, "feats.pkl"))
    rets3 = gan.reconstruct_dataset()
    np.testing.assert_array_equal(rets3["dev"][0], rets["dev"][0])
    # test_again forces recomputation; max_num changes the directory name
    gan.test_again = True
    gan.reconstruct_dataset()
    assert calls == [2, 2, 1, 2, 1, 2, 2]
    assert gan.rec_cache_dir("dev", max_num=100).endswith(os.path.join("recs_rr2_lr0.50000_iters3_num100", "dev"))


def _gloo_dataset_worker(rank, world, port, out_dir, ret):
    """reconstruct_dataset on every rank of a gloo group: batches sharded over the ranks, rank 0 owns the cache."""
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from defensegan_b200.models.gan import MnistDefenseGAN, RecCache
        gan = MnistDefenseGAN(test_mode=True, verbose=False, output_dir=out_dir)
        gan.initialized = True
        gan.rec_rr, gan.rec_lr, gan.rec_iters = 2, 0.5, 3
        shards = []

        def fake_reconstruct(x, z_init_val=None, out=None, z_row_offset=0, **kw):   # stand-in for the CUDA projector
            shards.append((int(x.shape[0]), int(z_row_offset)))
            out.copy_(x * 0.5)
            return out

        gan.reconstruct = fake_reconstruct
        rs = np.random.RandomState(0)
        data = {sp: (rs.randint(0, 256, size=(n, 28, 28, 1)).astype("uint8"), np.arange(n) % 10)
                for sp, n in (("train", 7), ("dev", 3), ("test", 4))}

        def gen(sp, bs=4):
            def g():
                x, y = data[sp]
                for i in range(0, len(x), bs):
                    yield x[i:i + bs], y[i:i + bs]
            return g

        stores = []
        orig_store = RecCache.store_batch
        RecCache.store_batch = lambda self, first, labels, recs: (stores.append(first), orig_store(self, first, labels, recs))
        gan.set_dataset_generators(train=gen("train"), dev=gen("dev"), test=gen("test"))
        rets = gan.reconstruct_dataset()
        ok = all(np.allclose(rets[sp][0], data[sp][0] / 255.0 * 0.5) and rets[sp][0].shape[0] == len(data[sp][0])
                 for sp in data)
        # batches of 4, 3 | 3 | 4 images split over two ranks: rank 0 takes the larger half; z0 rows start at
        # (first image of the shard) * rec_rr
        want = {0: [(2, 0), (2, 0), (2, 0), (2, 0)], 1: [(2, 4), (1, 4), (1, 4), (2, 4)]}[rank]
        ok = ok and shards == want and (len(stores) == 4) == (rank == 0)
        dist.barrier()                                   # rank 0's files are on disk
        shards.clear()
        rets2 = gan.reconstruct_dataset()               # second pass: rank 0 reports hits, nobody projects
        ok = ok and shards == [] and all(np.array_equal(rets2[sp][0], rets[sp][0]) for sp in data)
        ret[rank] = ok
    finally:
        dist.destroy_process_group()


def test_reconstruct_dataset_shards_batches_over_ranks_gloo_world2(tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    ret = ctx.Manager().dict()
    port = _free_port()
    procs = [ctx.Process(target=_gloo_dataset_worker, args=(r, 2, port, str(tmp_path), ret)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(180)
        assert p.exitcode == 0
    assert ret[0] and ret[1]


# ---------------------------------------------------------------------------------------------------
# f2: TensorFlow checkpoint-V2 bundle reader (no TensorFlow needed)
# ---------------------------------------------------------------------------------------------------
def _bundle_tensors():
    rs = np.random.RandomState(5)
    t = {"Generator.Input/Generator.Input.W": rs.randn(8, 32).astype("float32"),
         "Generator.Input/Generator.Input.b": rs.randn(32).astype("float32"),
         "Generator.2/Generator.2.Filters": rs.randn(5, 5, 4, 8).astype("float32"),
         "Generator.2/Generator.2.Filters/Adam": rs.randn(5, 5, 4, 8).astype("float32"),
         "Generator.2/Generator.2.Filters/Adam_1": rs.randn(5, 5, 4, 8).astype("float32"),
         "Discriminator.1/Discriminator.1.Filters": rs.randn(5, 5, 1, 4).astype("float32"),
         "global_step": np.asarray(20000, dtype="int64"),
         "beta1_power": np.asarray(0.5, dtype="float32")}
    for i in range(40):   # many similar names: exercises prefix compression and restart points
        t["Discriminator.%02d/Discriminator.%02d.Biases" % (i, i)] = rs.randn(3 + i).astype("float32")
    return t


def test_tf_bundle_roundtrip_prefix_compression_and_blocks(tmp_path):
    from defensegan_b200 import tf_bundle as B
    t = _bundle_tensors()
    for block_size in (262144, 64):          # one data block / many data blocks + a multi-entry index block
        prefix = str(tmp_path / ("bs%d" % block_size) / "GAN.model-20000")
        B.write_bundle(prefix, t, block_size=block_size)
        listed = B.list_bundle(prefix)
        assert list(listed) == sorted(t, key=lambda s: s.encode()) and listed["global_step"] == (np.dtype("<i8"), ())
        back = B.read_bundle(prefix)
        assert set(back) == set(t)
        for k in t:
            assert back[k].dtype == t[k].dtype and back[k].shape == t[k].shape and np.array_equal(back[k], t[k])
        gen = B.read_generator_variables(prefix)
        assert sorted(gen) == ["Generator.2/Generator.2.Filters", "Generator.Input/Generator.Input.W",
                               "Generator.Input/Generator.Input.b"]
        with pytest.raises(KeyError):
            B.read_bundle(prefix, ["nope"])


def test_tf_bundle_matches_independent_crc_and_proto_implementations():
    """CRC-32C, its masking and the TensorShapeProto wire format against TensorBoard's own implementations
    (the only TensorFlow-lineage code in this image)."""
    from defensegan_b200 import tf_bundle as B
    assert B.crc32c(b"123456789") == 0xE3069283            # CRC-32C check value (RFC 3720)
    assert B.crc32c(b"\x00" * 32) == 0x8A9136AA and B.crc32c(b"\xff" * 32) == 0x62A8AB43
    assert B.unmask_crc(B.mask_crc(0xDEADBEEF)) == 0xDEADBEEF
    tb = pytest.importorskip("tensorboard.compat.tensorflow_stub.pywrap_tensorflow")
    rs = np.random.RandomState(0)
    for n in (0, 1, 7, 4096, 10001):
        blob = rs.bytes(n)
        assert B.crc32c(blob) == tb.crc32c(blob)
        assert B.mask_crc(B.crc32c(blob)) == tb.masked_crc32c(blob)
    shape_pb2 = pytest.importorskip("tensorboard.compat.proto.tensor_shape_pb2")
    for shape in ((), (7,), (5, 5, 128, 256), (1, 0, 300)):
        msg = shape_pb2.TensorShapeProto()
        for d in shape:
            msg.dim.add().size = d
        assert B.encode_tensor_shape(shape) == msg.SerializeToString()
        assert B.parse_tensor_shape(msg.SerializeToString()) == tuple(shape)
        assert tuple(d.size for d in shape_pb2.TensorShapeProto.FromString(B.encode_tensor_shape(shape)).dim) == tuple(shape)
    types_pb2 = pytest.importorskip("tensorboard.compat.proto.types_pb2")
    for enum, dt in B._DTYPE_OF.items():
        name = types_pb2.DataType.Name(enum)
        assert name == {"<f4": "DT_FLOAT", "<f8": "DT_DOUBLE", "<i4": "DT_INT32", "|u1": "DT_UINT8", "<i2": "DT_INT16",
                        "|i1": "DT_INT8", "<i8": "DT_INT64", "|b1": "DT_BOOL", "<u2": "DT_UINT16", "<f2": "DT_HALF",
                        "<u4": "DT_UINT32", "<u8": "DT_UINT64"}[dt.str]


def test_tf_bundle_roundtrip_property(tmp_path):
    """Random names (shared prefixes, so prefix compression and restart points are hit), dtypes, ranks 0-4 and block
    sizes: write_bundle -> list_bundle / read_bundle returns the same arrays bit for bit, keys in sorted order."""
    hypothesis = pytest.importorskip("hypothesis")
    from hypothesis import given, settings, strategies as st
    from defensegan_b200 import tf_bundle as B
    dtypes = ["<f4", "<f8", "<i4", "<i8", "|u1", "<f2", "|b1"]
    names = st.text(alphabet="abG./_0123456789", min_size=1, max_size=24).map(lambda t: "Generator." + t)
    tensor = st.tuples(st.sampled_from(dtypes), st.lists(st.integers(0, 5), min_size=0, max_size=4), st.integers(0, 2 ** 31 - 1))
    counter = [0]

    @settings(max_examples=30, deadline=None)
    @given(st.dictionaries(names, tensor, min_size=1, max_size=12), st.sampled_from([64, 300, 4096, 262144]))
    def run(spec, block_size):
        counter[0] += 1
        prefix = str(tmp_path / ("case%d" % counter[0]) / "GAN.model-7")
        tensors = {}
        for name, (dt, shape, seed) in spec.items():
            rs = np.random.RandomState(seed)
            tensors[name] = (rs.randint(0, 255, size=shape) if dt != "|b1" else rs.randint(0, 2, size=shape)).astype(np.dtype(dt))
        B.write_bundle(prefix, tensors, block_size=block_size)
        listed = B.list_bundle(prefix)
        assert list(listed) == sorted(tensors)
        got = B.read_bundle(prefix)
        for name, want in tensors.items():
            assert got[name].dtype == want.dtype and got[name].shape == want.shape and np.array_equal(got[name], want)
            assert listed[name] == (want.dtype, want.shape)

    run()


def test_tf_bundle_detects_corruption(tmp_path):
    from defensegan_b200 import tf_bundle as B
    prefix = str(tmp_path / "GAN.model-1")
    B.write_bundle(prefix, {"Generator.Input/Generator.Input.b": np.arange(64, dtype="float32")})
    data = prefix + ".data-00000-of-00001"
    raw = bytearray(open(data, "rb").read())
    raw[10] ^= 0x40
    open(data, "wb").write(bytes(raw))
    with pytest.raises(ValueError, match="checksum"):
        B.read_bundle(prefix)
    assert B.read_bundle(prefix, verify_crc=False)["Generator.Input/Generator.Input.b"].shape == (64,)
    idx = bytearray(open(prefix + ".index", "rb").read())
    idx[3] ^= 0x01
    open(prefix + ".index", "wb").write(bytes(idx))
    with pytest.raises(ValueError):
        B.read_bundle(prefix)
    open(prefix + ".index", "wb").write(b"not a table")
    with pytest.raises(ValueError):
        B.list_bundle(prefix)


def test_load_generator_from_tf_checkpoint_dir(tmp_path):
    """models/gan.py:80-87: restore the Generator variables of the latest checkpoint in the model's dir."""
    from defensegan_b200.models.gan import MnistDefenseGAN
    from defensegan_b200 import tf_bundle as B
    from defensegan_b200.weights import init_generator_weights
    src = init_generator_weights("mnist", seed=7)
    ckpt = tmp_path / "gans" / "mnist"
    extra = {"Discriminator.1/Discriminator.1.Filters": np.zeros((5, 5, 1, 64), "float32"),
             "Generator.2/Generator.2.Filters/Adam": np.ones((5, 5, 128, 256), "float32"), "global_step": np.asarray(500, "int64")}
    B.write_bundle(str(ckpt / "GAN.model-0"), {k: v * 0 for k, v in src.items()})
    B.write_bundle(str(ckpt / "GAN.model-500"), dict(src, **extra))
    (ckpt / "checkpoint").write_text('model_checkpoint_path: "GAN.model-500"\nall_model_checkpoint_paths: "GAN.model-0"\n'
                                     'all_model_checkpoint_paths: "GAN.model-500"\n')
    assert B.latest_checkpoint(str(ckpt)).endswith("GAN.model-500")
    gan = MnistDefenseGAN(test_mode=True, verbose=False)
    assert gan.load_generator(str(ckpt)) is True
    for k, v in src.items():
        assert np.array_equal(gan.weights[k], v)
    (ckpt / "checkpoint").unlink()                       # no state file: highest step wins
    assert B.latest_checkpoint(str(ckpt)).endswith("GAN.model-500")
    out = gan.save_generator(str(tmp_path / "export"), fmt="tf", global_step=3)
    gan2 = MnistDefenseGAN(test_mode=True, verbose=False)
    assert gan2.load_generator(str(tmp_path / "export")) is True and out.endswith("GAN.model-3")
    assert all(np.array_equal(gan2.weights[k], v) for k, v in src.items())
    assert MnistDefenseGAN(test_mode=True, verbose=False).load_generator(str(tmp_path / "empty")) is False


# ---------------------------------------------------------------------------------------------------
# tensor-core schedule planner (host code of the CUDA library; needs no GPU)
# ---------------------------------------------------------------------------------------------------
def _check_plans(arch, n_rows, n_pairs=66, net_dim=64, mutate=0, use_bn=0):
    import ctypes
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_check_plans.restype = ctypes.c_int
    lib.dgan_debug_check_plans.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.dgan_last_error.restype = ctypes.c_char_p
    desc = _native.dgan_desc(_native.ABI_VERSION, 0 if arch == "mnist" else 1, 128, net_dim, use_bn, 1)
    rc = lib.dgan_debug_check_plans(ctypes.byref(desc), n_rows, n_pairs, mutate)
    return rc, (lib.dgan_last_error() or b"").decode()


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_schedule_plans_are_valid_for_many_batch_sizes(arch):
    """Every plan the library would upload - window tiling, LPT assignment, step streams, ring offsets and
    dependency distances, merged-N groups - is re-derived and checked by tc2_check_plan: exact coverage of the pair
    tables, first-MMA flags, canonical accumulation order (=> batch-size / sharding invariance), ring safety."""
    for n_rows in (1, 10, 256, 500, 1280, 2560, 5000):           # B*R; 2560 = BASELINE configs[1], 1280 = CelebA C4
        rc, msg = _check_plans(arch, n_rows)
        assert rc == 0, "n_rows=%d: %s" % (n_rows, msg)
    for n_pairs in (1, 3, 37, 66):                               # fewer SMs available (smaller parts, MIG slices)
        rc, msg = _check_plans(arch, 2560 if arch == "mnist" else 640, n_pairs=n_pairs)
        assert rc == 0, "n_pairs=%d: %s" % (n_pairs, msg)


def test_schedule_plans_are_valid_for_random_sizes_and_sm_counts():
    """Any (latent rows, CTA pairs, net_dim) a caller or a smaller part could present: ragged batches of model_eval_gan,
    MIG slices, half-width generators."""
    pytest.importorskip("hypothesis")
    from hypothesis import given, settings, strategies as st

    @settings(max_examples=40, deadline=None)
    @given(st.sampled_from(["mnist", "celeba"]), st.integers(1, 3000), st.integers(1, 74), st.sampled_from([64, 64, 64, 32]),
           st.sampled_from([0, 0, 1]))
    def run(arch, n_rows, n_pairs, net_dim, use_bn):
        rc, msg = _check_plans(arch, n_rows, n_pairs=n_pairs, net_dim=net_dim, use_bn=use_bn)
        # a geometry the tensor-core path does not serve must be refused by name, never planned wrongly
        assert rc == 0 or "unsupported" in msg.lower(), (arch, n_rows, n_pairs, net_dim, use_bn, msg)

    run()


def test_schedule_planning_stays_bounded_for_large_batches():
    """configs[4] on ONE GPU (4096 images x 10 restarts = 160 row pairs) and a 1536-image CelebA batch: the assignment
    refinement is quadratic in the items per CTA pair and runs on a budget of candidate evaluations (TC2_REFINE_BUDGET,
    never reached by the benchmarked sizes), so planning - which dgan_workspace_bytes does on first sight of a batch
    size - takes seconds, and the plans still pass the validator.  (Unbounded, the CelebA case took 40 s, larger ones
    minutes.)"""
    import time
    for arch, n_rows in (("mnist", 40960), ("celeba", 15360)):
        t0 = time.time()
        rc, msg = _check_plans(arch, n_rows)
        assert rc == 0, "%s n_rows=%d: %s" % (arch, n_rows, msg)
        assert time.time() - t0 < 60.0, (arch, n_rows, time.time() - t0)


@pytest.mark.parametrize("arch", ["mnist", "celeba"])
def test_schedule_plans_with_batchnorm_geometry(arch):
    """use_bn=True on the tensor-core path: MNIST's Generator.2 then lives on the 8x8 raster (BN2 sees the cropped outputs
    too), so Generator.3's backward has output pixels that receive nothing - they must still be written (exact zeros
    through the zero weight tile) and no window may come without a step (its epilogue would wait for ever)."""
    for n_rows in (4, 256, 2560):
        rc, msg = _check_plans(arch, n_rows, use_bn=1)
        assert rc == 0, "n_rows=%d: %s" % (n_rows, msg)


def test_plan_statistics_entry_point():
    """tools/plan_stats.py's entry point: one line per layer-direction with the staged bytes and the balance of the
    assignment; configs[1] stages < 1.9 GB per L-step and no big layer's busiest CTA pair exceeds the mean by 12 %."""
    import ctypes
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_plan_stats.restype = ctypes.c_int
    lib.dgan_debug_plan_stats.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    desc = _native.dgan_desc(_native.ABI_VERSION, 0, 128, 64, 0, 1)
    buf = ctypes.create_string_buffer(1 << 16)
    assert lib.dgan_debug_plan_stats(ctypes.byref(desc), 2560, 66, buf, len(buf)) > 0
    rows = [l.split(" | ") for l in buf.value.decode().strip().splitlines()[1:]]
    by = {r[0]: r for r in rows}
    assert float(by["total staged MB per L-step"][1]) < 1900.0
    for name in ("Generator.2.fwd", "Generator.2.bwd", "Generator.3.fwd", "Generator.3.bwd"):
        assert float(by[name][9]) < 1.12, (name, by[name])


# The epilogue and output type each layer-direction of the fp16 path launches with.  With BatchNorm after a layer
# (use_bn: the Linear, Generator.2 and Generator.3) its forward stores fp32 pre-activations without the ReLU, and the
# backward into its output applies no ReLU mask: the BN backward does both.
_EPILOGUES = {           # direction: MNIST, MNIST + BN, CelebA, CelebA + BN (None: no such direction)
    "Linear.fwd": ("bias_relu/f16", "bias/f32", "bias_relu/f16", "bias/f32"),
    "Linear.bwd": ("none/f32", "none/f32", "none/f32", "none/f32"),
    "Generator.2.fwd": ("bias_relu/f16", "bias/f32", "bias_relu/f16", "bias/f32"),
    "Generator.2.bwd": ("mask/f16", "none/f16", "mask/f16", "none/f16"),
    "Generator.3.fwd": ("bias_relu/f16", "bias/f32", "bias_relu/f16", "bias/f32"),
    "Generator.3.bwd": ("mask/f16", "none/f16", "mask/f16", "none/f16"),
    "Generator.5.fwd": (None, None, "bias/f16", "bias/f16"),
    "Generator.5.bwd": (None, None, "mask/f16", "none/f16"),
    "last.fwd": ("final_sigmoid/f16", "final_sigmoid/f16", "final_tanh/f16", "final_tanh/f16"),
    "last.bwd": ("mask/f16", "none/f16", "none/f16", "none/f16"),
}


@pytest.mark.parametrize("arch,use_bn", [("mnist", 0), ("mnist", 1), ("celeba", 0), ("celeba", 1)])
def test_plans_are_made_for_the_epilogue_each_direction_launches_with(arch, use_bn):
    """The epilogue and output type set a plan's instantiation and ring size, so the plans the validator checks and the
    statistics describe must be made for the ones the launch uses.  The statistics name them in their last column."""
    import ctypes
    from defensegan_b200 import _native
    lib = _native.load_library()
    lib.dgan_debug_plan_stats.restype = ctypes.c_int
    lib.dgan_debug_plan_stats.argtypes = [ctypes.POINTER(_native.dgan_desc), ctypes.c_int, ctypes.c_int, ctypes.c_char_p, ctypes.c_int]
    desc = _native.dgan_desc(_native.ABI_VERSION, _native.ARCH_IDS[arch], 128, 64, use_bn, _native.PRECISIONS["fp16"])
    buf = ctypes.create_string_buffer(1 << 16)
    assert lib.dgan_debug_plan_stats(ctypes.byref(desc), 256, 66, buf, len(buf)) > 0
    lines = [l.split(" | ") for l in buf.value.decode().strip().splitlines()]
    assert len(lines[0]) == 16 and lines[0][15] == "epilogue/output", lines[0]
    col = 2 * (arch == "celeba") + use_bn
    want = {name: v[col] for name, v in _EPILOGUES.items() if v[col] is not None}
    assert [(r[0], r[15]) for r in lines[1:-1]] == list(want.items())     # in launch order


def test_schedule_validator_rejects_damaged_plans():
    """The validator is not vacuous: nine single faults injected into a valid plan (wrong first-MMA flag, accumulator,
    staged weight tile, input pixel, k-chunk, lost epilogue item, unsafe ring dependencies, region outside the ring,
    steps out of canonical order) are each reported."""
    assert _check_plans("mnist", 2560)[0] == 0
    seen = set()
    for mutate in range(1, 10):
        rc, msg = _check_plans("mnist", 2560, mutate=mutate)
        assert rc != 0 and msg.startswith("Generator.3.fwd:"), (mutate, rc, msg)
        seen.add(msg)
    assert len(seen) >= 5, seen          # different faults are told apart
