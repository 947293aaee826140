"""Host-side mirror of the reference's `models/gan.py` model classes for the projection loop.

Same class names, attribute names, defaults, argument meaning and error behaviour as
`DefenseGANBase` and its dataset subclasses (reference models/gan.py:39-135,333-449,649-765),
with the TF1 graph machinery replaced by eager calls into the native sm_90a library:

    gan = MnistDefenseGAN(cfg=cfg, test_mode=True)
    gan.load_generator()                      # reference models/gan.py:86-87
    gan.rec_rr, gan.rec_lr, gan.rec_iters = 10, 10.0, 200   # callers set these (blackbox.py:649-658)
    x_hat = gan.reconstruct(images)           # torch CUDA tensor [B,H,W,C] in, same shape out

Graph-mode -> eager mapping (SURVEY section 8b): `images` is a float32 CUDA tensor (NHWC,
already input-transformed) instead of a symbolic placeholder; the result is a detached tensor
(the reference graph has no gradient path from `images` to the output either, SURVEY F11);
`batch_size`, `back_prop` and `reconstructor_id` are accepted for signature compatibility -
any batch size works (superset of the reference's static-shape graph, SURVEY F10).
"""
from __future__ import annotations

import os
import pickle
import time
from typing import Callable, Dict, Iterable, Optional

import numpy as np
import torch

from .. import _native
from ..operators import ConvOperator
from .. import tf_bundle as _tf_bundle
from .. import weights as _weights
from ..utils.config import load_config, packaged_cfg_path

__all__ = ["RecCache", "DefenseGANBase", "MnistDefenseGAN", "FmnistDefenseDefenseGAN", "CelebADefenseGAN", "dataset_gan_dict"]

_NOT_GIVEN = object()      # reconstruct_measured's prune when the caller passed none (None means "do not prune")


class RecCache(object):
    """On-disk cache of one split's reconstructions, in the reference's layout (models/gan.py:466-478,503-507) so that
    its consumers (blackbox.py:249-259,294-329) keep working:

        <dir>/feats.pkl                         the whole split, one pickled array (written by save_recs)
        <dir>/pickles/rec_{index:07d}_l{label}.pkl   one pickled [H,W,C] array per image

    `index` = position of the image in the split.  Unreadable or missing entries simply count as misses (the reference
    tolerates broken cache files the same way, gan.py:486-496,526-534)."""

    def __init__(self, directory, reuse=True):
        self.directory = directory
        self.reuse = reuse
        self.pickle_dir = os.path.join(directory, 'pickles')
        os.makedirs(self.pickle_dir, exist_ok=True)

    @property
    def split_path(self):
        return os.path.join(self.directory, 'feats.pkl')

    def image_path(self, index, label):
        return os.path.join(self.pickle_dir, 'rec_{:07d}_l{}.pkl'.format(int(index), label))

    @staticmethod
    def _read(path):
        try:
            with open(path, 'rb') as f:
                return pickle.load(f)
        except Exception:
            return None

    def load_split(self):
        return self._read(self.split_path) if self.reuse else None

    def load_batch(self, first_index, labels):
        """The batch's reconstructions if EVERY image of it is cached, else None."""
        if not self.reuse:
            return None
        out = []
        for i, label in enumerate(labels):
            r = self._read(self.image_path(first_index + i, label))
            if r is None:
                return None
            out.append(r)
        return np.stack(out) if out else None

    def store_batch(self, first_index, labels, recs):
        for i, label in enumerate(labels):
            with open(self.image_path(first_index + i, label), 'wb') as f:
                pickle.dump(recs[i], f, protocol=pickle.HIGHEST_PROTOCOL)

    def store_split(self, recs):
        with open(self.split_path, 'wb') as f:
            pickle.dump(recs, f, pickle.HIGHEST_PROTOCOL)


class DefenseGANBase(object):
    """Holds the hyper-parameters, binds the generator and exposes reconstruct()."""

    _dataset_default = None
    _image_dim_default = [None, None, None]

    def __init__(self, cfg=None, test_mode=False, verbose=True, **args):
        # defaults of reference models/gan.py:50-69 (those the projection loop reads)
        self.dataset_name = self._dataset_default
        self.batch_size = 32
        self.use_bn = True                 # class default; every shipped cfg sets USE_BN False (SURVEY F1)
        self.test_batch_size = 20
        self.mode = "gp-wgan"
        self.latent_dim = None
        self.net_dim = None
        self.input_transform_type = 0
        self.debug = False
        self.rec_iters = 200
        self.image_dim = list(self._image_dim_default)
        self.rec_rr = 10
        self.rec_lr = 10.0
        self.test_again = False
        self.attribute = "gender"
        self.output_dir = "output"
        # additions of this implementation
        self.precision = "fp32"            # 'fp32' (CUDA-core, reference arithmetic) | 'fp16' (wgmma operands)
        self.rec_momentum = 0.7            # tf.train.MomentumOptimizer(momentum=0.7), models/gan.py:389-391
        self.rec_decay_lr = False          # the reference's decay is dead code (SURVEY F3); True = intended schedule
        self.rec_prune = None              # restart pruning: [(iter, keep), ...] (cfg REC_PRUNE); None = every restart to the end
        self.rec_optimizer = "momentum"    # update of z: "momentum" (the reference's) | "adam" (cfg REC_OPTIMIZER)
        self.rec_adam_betas = (0.9, 0.999)  # Adam's (beta1, beta2) (cfg REC_ADAM_BETAS), read with rec_optimizer "adam"
        self.rec_adam_eps = 1e-8           # Adam's eps (cfg REC_ADAM_EPS)
        self.rec_huber_delta = None        # data term: None = squared error (the reference's) | Huber delta > 0 (cfg REC_HUBER_DELTA)
        self.rec_z_prior = None            # latent prior: None = none (the reference's) | lambda >= 0 of D + lambda ||z||^2 (cfg REC_Z_PRIOR)
        self.rec_sparse_dev = None         # sparse deviations: None = none (the reference's) | (l1, step) of G(z) + nu (cfg REC_SPARSE_DEV)
        self.seed = 11241990               # callers use tf.set_random_seed(11241990) (blackbox.py:464)

        self.test_mode = test_mode
        self.verbose = verbose
        self.is_training = not test_mode
        self.initialized = False
        self._set_attr(cfg, args)
        if self.latent_dim is None:
            self.latent_dim = 128
        if self.net_dim is None:
            self.net_dim = 64
        self._set_checkpoint_dir()
        self._build()
        self._native = None
        self._native_key = None
        self._call_counter = 0
        # TF creates the variables with their random initial values at graph construction;
        # load_generator() later overwrites them from a checkpoint.
        self.weights = _weights.init_generator_weights(self.arch, seed=self.seed, latent_dim=self.latent_dim,
                                                       net_dim=self.net_dim, use_bn=bool(self.use_bn))

    # -- configuration (reference models/base_model.py:120-148) ------------------------------
    def _set_attr(self, cfg, args):
        if cfg is None:
            # no cfg given: the packaged copy of the dataset's yml over default.yml
            ds = args.get("dataset_name", self.dataset_name)
            cfg = load_config(packaged_cfg_path(ds)) if ds is not None else None
        elif isinstance(cfg, str):
            cfg = load_config(cfg)
        self.cfg = cfg
        known = [k for k in self.__dict__.keys() if not k.startswith("_")]
        for attr in known:
            val = None
            if cfg is not None:
                if attr.upper() in cfg:
                    val = cfg[attr.upper()]
                elif attr in cfg:
                    val = cfg[attr]
            if attr in args:
                val = args[attr]
            if val is not None:
                setattr(self, attr, val)
        unknown = [k for k in args if k not in known]
        if unknown:
            raise TypeError("unexpected keyword argument(s): %s" % ", ".join(sorted(unknown)))
        if self.image_dim is not None:
            self.image_dim = [int(v) if v is not None else None for v in self.image_dim]

    def _set_checkpoint_dir(self):
        """Where the model's snapshots live (reference models/base_model.py:197-232, test-mode branch): the directory
        of an experiment's own `cfg.yml`, else `<output_dir>/<cfg path relative to experiments/cfgs, without .yml>`
        (`experiments/cfgs/gans/mnist.yml` -> `output/gans/mnist`).  The packaged cfgs map the same way."""
        cfg_file = str((self.cfg or {}).get('cfg_path', '') or '')
        if os.path.basename(cfg_file) == 'cfg.yml':
            self.checkpoint_dir = os.path.dirname(cfg_file)
            return
        rel = None
        norm = cfg_file.replace(os.sep, '/')
        for marker in ('experiments/cfgs/', '/cfgs/'):
            if marker in norm:
                rel = norm.split(marker)[-1]
                break
        if rel is None:
            rel = os.path.join('gans', str(self.dataset_name))
        if rel.endswith('.yml'):
            rel = rel[:-4]
        self.checkpoint_dir = os.path.join(str(self.output_dir), rel)

    def _build(self):
        # reference models/gan.py:101-105
        assert (self.batch_size % self.rec_rr) == 0, 'Batch size should be divisable by random restart'
        self.test_batch_size = self.batch_size
        self.arch = _weights.canonical_arch(self.dataset_name)
        expect = list(_weights.IMAGE_DIMS[self.arch])
        if self.image_dim is None or any(v is None for v in self.image_dim):
            self.image_dim = expect
        if list(self.image_dim) != expect:
            raise ValueError("image_dim %s does not match the %s generator (%s)" % (self.image_dim, self.arch, expect))

    # -- weights -----------------------------------------------------------------------------
    def set_generator_weights(self, weights: Dict[str, np.ndarray]) -> None:
        """Install generator weights (names per the tflib.param registry, see weights.py)."""
        _weights.validate_weights(self.arch, weights, self.latent_dim, self.net_dim, bool(self.use_bn))
        self.weights = {k: np.asarray(v, dtype=np.float32) for k, v in weights.items()}
        self._drop_native()
        self.initialized = True

    def load_generator(self, ckpt_path=None):
        """Restore the generator (reference models/gan.py:80-87 -> base_model.py:294-335).
        `ckpt_path` is the model's checkpoint dir (default), a `generator.npz`, or a TF checkpoint prefix
        (`.../GAN.model-20000`).  A directory is searched for `generator.npz` first, then for the latest
        TensorFlow checkpoint-V2 bundle (`checkpoint` state file / `*.index`), which is read without
        TensorFlow by `defensegan_b200.tf_bundle` - only the `Generator*` variables, as the reference does.
        Returns False (and keeps the random-init weights, like the reference's failed restore,
        base_model.py:312-317) when nothing is found."""
        path = ckpt_path if ckpt_path is not None else self.checkpoint_dir
        for suffix in ('.index', '.meta'):                       # a bundle's file name instead of its prefix
            if path.endswith(suffix):
                path = path[:-len(suffix)]
        if '.data-' in os.path.basename(path):
            path = path[:path.rindex('.data-')]
        npz, prefix = None, None
        if os.path.isdir(path):
            if os.path.isfile(os.path.join(path, "generator.npz")):
                npz = os.path.join(path, "generator.npz")
            else:
                prefix = _tf_bundle.latest_checkpoint(path)
        elif os.path.isfile(path):
            npz = path
        elif os.path.isfile(path + ".index"):
            prefix = path
        if npz is not None:
            self.set_generator_weights(_weights.load_npz(npz))
        elif prefix is not None:
            self.set_generator_weights(_tf_bundle.read_generator_variables(prefix))
        else:
            msg = "[-] No generator checkpoint found at {}; keeping random-init weights".format(path)
            if self.test_mode:
                # the reference's callers ignore the return value (blackbox.py:640-642): projecting onto an untrained
                # generator must not pass silently
                import warnings
                warnings.warn(msg, RuntimeWarning, stacklevel=2)
            elif self.verbose:
                print(msg)
            return False
        if self.verbose:
            print("[*] Generator restored from {}".format(npz or prefix))
        return True

    def save_generator(self, ckpt_path=None, fmt="npz", global_step=0):
        """`fmt="npz"`: `generator.npz`; `fmt="tf"`: a TensorFlow checkpoint-V2 bundle `GAN.model-<step>` plus the
        `checkpoint` state file, the layout of the reference's saver (base_model.py:383-395)."""
        path = ckpt_path if ckpt_path is not None else self.checkpoint_dir
        if fmt == "tf":
            os.makedirs(path, exist_ok=True)
            name = "GAN.model-%d" % int(global_step)
            _tf_bundle.write_bundle(os.path.join(path, name), dict(self.weights))
            with open(os.path.join(path, "checkpoint"), "w") as f:
                f.write('model_checkpoint_path: "%s"\nall_model_checkpoint_paths: "%s"\n' % (name, name))
            return os.path.join(path, name)
        if not path.endswith(".npz"):
            os.makedirs(path, exist_ok=True)
            path = os.path.join(path, "generator.npz")
        _weights.save_npz(path, self.weights)
        return path

    # -- native handle -------------------------------------------------------------------------
    def _drop_native(self):
        if getattr(self, "_native", None) is not None:
            self._native.close()
        self._native = None
        self._native_key = None

    def _get_native(self, device) -> "_native.NativeGenerator":
        key = (str(device), self.precision, int(self.latent_dim), int(self.net_dim), bool(self.use_bn))
        if self._native is None or self._native_key != key:
            self._drop_native()
            ordered = _weights.validate_weights(self.arch, self.weights, self.latent_dim, self.net_dim, bool(self.use_bn))
            tensors = [torch.as_tensor(np.ascontiguousarray(w), dtype=torch.float32).to(device) for w in ordered]
            self._native = _native.NativeGenerator(self.arch, tensors, latent_dim=self.latent_dim, net_dim=self.net_dim,
                                                   use_bn=bool(self.use_bn), precision=self.precision, device=device)
            self._native_key = key
        return self._native

    # -- the hot path ------------------------------------------------------------------------------
    def input_transform(self, X):
        raise NotImplementedError

    def generator_fn(self, z=None, is_training=False):
        """G(z) (reference models/gan.py:657-665,726-735): z [N, latent] -> images [N,H,W,C].
        Differentiable in z like the reference's graph: when z requires grad (and grad mode is on) the result has a
        grad_fn whose backward is the native vector-Jacobian product; otherwise it is a plain tensor."""
        if z is None:
            raise ValueError("z must be given (sampling inside generator_fn is a training-time feature)")
        z = self._as_cuda(z)
        return _native.generator(self._get_native(z.device), z)

    def generator_jacobian(self, z):
        """dG/dz at each row of z [N, latent] as [N,H,W,C,latent] (NativeGenerator.jacobian: forward-mode products with
        identity tangents).  Its columns span the tangent space of the range of G at G(z).  Refused with use_bn."""
        z = self._as_cuda(z)
        return self._get_native(z.device).jacobian(z)

    @staticmethod
    def _as_cuda(t):
        if isinstance(t, np.ndarray):
            t = torch.from_numpy(np.ascontiguousarray(t))
        if not isinstance(t, torch.Tensor):
            raise TypeError("expected a torch.Tensor or numpy array")
        if not t.is_cuda:
            if not torch.cuda.is_available():
                raise RuntimeError("defensegan_b200 needs a CUDA (sm_90) device; there is no CPU fallback")
            t = t.cuda(non_blocking=True)
        return t.to(torch.float32)

    def _next_seed(self, reconstructor_id=0):
        """Philox key of the next call's z0 stream (fresh per call, like re-running the initialiser, gan_defense.py:119)."""
        self._call_counter += 1
        return (int(self.seed) * 1000003 + int(reconstructor_id) * 7919 + self._call_counter) & (2 ** 63 - 1)

    def reconstruct(self, images, batch_size=None, back_prop=True, reconstructor_id=0, z_init_val=None,
                    return_aux=False, out=None, z_row_offset=0, pixel_weights=None, deviation_out=None):
        """Defense-GAN projection of `images` onto the generator's range (reference
        models/gan.py:333-449): rec_rr restarts x rec_iters momentum-GD steps on
        ||G(z) - x||^2, returns G(z) of the min-loss restart.  Hyper-parameters are read from the
        object at call time.  Fresh z0 ~ N(0, 1/latent_dim) and zero momentum on every call
        (utils/gan_defense.py:119) unless `z_init_val` [B*rec_rr, latent_dim] is given
        (models/gan.py:395-397).  `z_row_offset` (sharded callers only): index of the first latent row of `images`
        in the call's z0 stream, so that a batch split over several GPUs draws what one GPU would.

        `pixel_weights` (an extension; the reference has none): a tensor or array that broadcasts to the images' shape,
        with finite values in [0, 1], to fit G(z) to part of each image - occluded or missing pixels (weight 0), pixels a
        detector flagged as corrupted, per-channel or per-region weighting.  The R restarts of an image share its weights.
        Each restart minimises (1/HWC) sum_p w_p (G(z)_p - x_p)^2: the normaliser stays H*W*C, so rec_lr means what it
        means unweighted, and weights covering a fraction f of the pixels give gradients about f times smaller (there is
        no renormalisation).  The returned loss and the arg-min restart use the weighted loss; an image whose weights are
        all 0 keeps its z0 and restart 0 is chosen.  With weights of 1 the result is bit-identical to the unweighted
        call.  The weights are checked before any native call - a ValueError for non-finite values or values outside
        [0, 1] - at the cost of one device reduction and one host read, on the weighted path only.

        `rec_prune` (an extension, read at call time; None by default): a list of (iter, keep) pairs,
        1 <= iter_1 < iter_2 < ... <= rec_iters - 1 and rec_rr >= keep_1 >= keep_2 >= ... >= 1.  From iteration iter_k on,
        each image runs only its keep_k restarts of lowest loss at iteration iter_k - 1 (ties: the lower restart index;
        NaN last); the survivors follow exactly the trajectories they would follow unpruned, and the arg-min picks among
        the last survivors (`return_aux`'s restart is the original index).  It cuts the row-steps of a call, at the risk of
        dropping a restart that would have won.  The schedule is checked before any native call (a ValueError naming the
        bad point), and refused with use_bn, whose batch statistics couple the restarts.

        `rec_optimizer` (an extension, read at call time; "momentum" by default, the reference's
        MomentumOptimizer(rec_lr, rec_momentum)): "adam" updates z with Adam, rec_adam_betas = (beta1, beta2) and
        rec_adam_eps, with m and s reset on every call and bias correction at step k = t + 1; rec_momentum is then
        ignored.  Adam's rec_lr is a step in z units (each coordinate moves by about rec_lr per step early on), so the
        reference's rec_lr = 10.0 does not carry over: choose it for the problem.  It combines with pixel_weights and
        rec_prune.  The values are checked before any native call (a ValueError naming the bad value).

        `rec_huber_delta` (an extension, read at call time; None by default, the reference's squared error): a delta > 0
        (+inf allowed) replaces the squared error by the Huber loss, quadratic for |G(z)_p - x_p| <= delta and linear
        beyond, so a few badly wrong pixels - impulse noise, dead pixels, an occluder whose place is not known - pull the
        fit much less; pixel_weights would need to know where they are.  The loss stays (1/HWC) sum_p w_p rho(d_p) with
        rho = 2 huber_loss, so delta = +inf, or delta >= 2 on images in the generator's output range, gives the squared
        error's bits.  With momentum the gradient of clipped residuals shrinks with delta, so rec_lr has to grow as delta
        falls; with rec_optimizer "adam" it does not.  It combines with pixel_weights, rec_prune and Adam, and is checked
        before any native call (a ValueError naming the bad value).

        `rec_z_prior` (an extension, read at call time; None by default, the reference's loss alone): a lambda >= 0 adds a
        Gaussian prior on z, so each restart minimises J = D + lambda ||z||^2 with D the data term above.  It keeps z where
        the generator was trained, so G(z) cannot fit noise or an adversarial perturbation with a latent of a norm the
        generator never saw.  D keeps its 1/HWC normaliser, so lambda is relative to the mean loss: the lambda of a
        formulation on the unnormalised sum does not carry over.  The returned loss is J (the detection statistic then
        includes the prior), the chosen restart is J's arg-min and rec_prune ranks by J.  lambda = 0 gives the bits of
        the call without it.  It combines with pixel_weights, rec_prune, Adam and rec_huber_delta, and is checked before
        any native call (a ValueError naming the bad value).

        `rec_sparse_dev` (an extension, read at call time; None by default, the reference's range projection alone): an
        (l1, step) pair with both >= 0 fits G(z) + nu, with nu a per-pixel deviation under an l1 penalty (Sparse-Gen,
        Dhar, Grover and Ermon 2018): each restart minimises D(G(z) + nu) [+ lambda ||z||^2] + l1 ||nu||_1, nu taking an
        ISTA step of size step * H*W*C / 2 each iteration.  A few pixels the generator cannot produce - an occluder, dead
        or saturated pixels, impulse noise, a patch - then go into nu instead of dragging z to a wrong latent.  The
        returned image is still G(z) of the chosen restart (the defense's output); `deviation_out` (a [B,H,W,C] float32
        CUDA tensor) receives that restart's nu, a per-pixel map of where the input left the generator's range.  step = 1
        on the squared error moves nu to its exact minimiser each step, counting residuals beyond l1 * H*W*C / 2 as
        deviations.  The returned loss is J with the l1 term, the arg-min and rec_prune rank by it.  It combines with
        pixel_weights, rec_prune, Adam, rec_huber_delta and rec_z_prior, and is checked before any native call (a
        ValueError naming the bad value).  The image loss then runs in the measured loop rather than the fused one, so
        it costs more per step."""
        prune = self._prune_schedule()
        adam = self._adam_params()
        huber = self._huber_delta()
        prior = self._z_prior()
        sdev = self._sparse_dev(deviation_out)
        x = self._as_cuda(images)
        if x.dim() != 4 or list(x.shape[1:]) != list(self.image_dim):
            raise ValueError("images must be [B,%d,%d,%d], got %s" % (tuple(self.image_dim) + (tuple(x.shape),)))
        if batch_size is not None and int(batch_size) != x.shape[0]:
            raise ValueError("batch_size (%d) does not match images.shape[0] (%d)" % (int(batch_size), x.shape[0]))
        pw = self._pixel_weights(pixel_weights, x) if pixel_weights is not None else None
        z0 = self._as_cuda(z_init_val) if z_init_val is not None else None
        native = self._get_native(x.device)
        self.last_seed = seed = self._next_seed(reconstructor_id)
        kw = {} if pw is None else {"pixel_weights": pw}
        if prune is not None:
            kw["prune"] = prune
        kw.update(self._option_kwargs(adam, huber, prior, sdev, deviation_out))
        res = native.reconstruct(x, int(self.rec_rr), int(self.rec_iters), float(self.rec_lr), z_init_val=z0, seed=seed,
                                 momentum=float(self.rec_momentum), decay_lr=bool(self.rec_decay_lr), out=out,
                                 return_aux=return_aux, z_row_offset=int(z_row_offset), **kw)
        return res

    @staticmethod
    def _option_kwargs(adam, huber, prior, sdev, deviation_out):
        """The native keyword arguments of the checked options that are set: an option left unset is not passed, so the
        call reaches the native layer as it did before that option existed."""
        kw = {} if adam is None else {"adam": adam}
        if huber is not None:
            kw["huber_delta"] = huber
        if prior is not None:
            kw["z_prior"] = prior
        if sdev is not None:
            kw["sparse_dev"] = sdev
            kw["deviation_out"] = deviation_out
        return kw

    def _prune_schedule(self):
        """`rec_prune` checked against rec_rr and rec_iters (None when unset); ValueError before any native call."""
        if self.rec_prune is None:
            return None
        if bool(self.use_bn):
            raise ValueError("rec_prune is not supported with use_bn: the batch statistics couple the restarts, so "
                             "dropping some would change the others' trajectories")
        return _native.check_prune_schedule(self.rec_prune, int(self.rec_rr), int(self.rec_iters))

    def _adam_params(self):
        """None for rec_optimizer "momentum", else Adam's (beta1, beta2, eps) from rec_adam_betas and rec_adam_eps,
        checked; ValueError naming the bad value before any native call."""
        opt = self.rec_optimizer
        if opt not in ("momentum", "adam"):
            raise ValueError("rec_optimizer = %r: expected 'momentum' or 'adam'" % (opt,))
        if opt == "momentum":
            return None
        betas = self.rec_adam_betas
        try:
            betas = tuple(betas)
        except TypeError:
            raise ValueError("rec_adam_betas = %r: expected a pair (beta1, beta2)" % (betas,)) from None
        if len(betas) != 2:
            raise ValueError("rec_adam_betas = %r: expected a pair (beta1, beta2)" % (betas,))
        return _native.check_adam_params((betas[0], betas[1], self.rec_adam_eps))

    def _huber_delta(self):
        """`rec_huber_delta` checked (None when unset): a float > 0, +inf allowed; ValueError before any native call."""
        if self.rec_huber_delta is None:
            return None
        try:
            return _native.check_huber_delta(self.rec_huber_delta)
        except ValueError as e:
            raise ValueError("rec_huber_delta: %s" % e) from None

    def _z_prior(self):
        """`rec_z_prior` checked (None when unset): a finite float >= 0; ValueError before any native call."""
        if self.rec_z_prior is None:
            return None
        try:
            return _native.check_z_prior(self.rec_z_prior)
        except ValueError as e:
            raise ValueError("rec_z_prior: %s" % e) from None

    def _sparse_dev(self, deviation_out=None):
        """`rec_sparse_dev` checked (None when unset): an (l1, step) pair of finite floats >= 0; ValueError before any
        native call, also for a deviation_out given without it."""
        if self.rec_sparse_dev is None:
            if deviation_out is not None:
                raise ValueError("deviation_out needs rec_sparse_dev: without deviations there is nothing to return")
            return None
        try:
            return _native.check_sparse_dev(self.rec_sparse_dev)
        except ValueError as e:
            raise ValueError("rec_sparse_dev: %s" % e) from None

    def reconstruct_measured(self, measurements, operator, batch_size=None, z_init_val=None, return_aux=False, out=None,
                             z_row_offset=0, prune=_NOT_GIVEN, deviation_out=None):
        """Projection onto the generator's range from linear measurements (an extension; the reference has none), for
        images that are not held themselves but observed as y = A x: a low-resolution or blurred copy, a
        compressed-sensing sketch.  `operator` A is [m, H*W*C] (a tensor or array; columns in NHWC pixel order,
        1 <= m <= H*W*C), one for every image and restart; `measurements` y is [B, m].  The R restarts of image i share
        y[i], and each minimises (1/m) ||A G(z) - y[i]||^2: the normaliser is m, so A = I gives the loss of `reconstruct`
        and rec_lr keeps its meaning.  rec_rr, rec_iters, rec_lr, the momentum and decay_lr are read from the object at
        call time, and z0 is drawn as in `reconstruct` (the same seed gives the same z0) unless `z_init_val`
        [B*rec_rr, latent_dim] is given.  Returns G(z) [B, H, W, C] of the restart with the lowest measured loss (with
        return_aux also that loss [B] and the restart [B]).  Shapes and finiteness are checked before any native call -
        a ValueError that names the bad input - at the cost of one device reduction and one host read.

        `operator` may also be a torch sparse tensor, COO (coalesced: duplicates summed) or CSR: the same semantics as the
        dense matrix it represents, at a cost set by its non-zeros - a block average, a blur kernel or pixel subsampling
        have a few non-zeros per row.  A CSR operator is checked too (2-D, not batched or hybrid, crow_indices rising
        from 0 to nnz, column indices in range and strictly ascending within each row).  On fp32 the result is
        bit-identical to the dense call on the same matrix; on fp16 a sparse operator is applied in fp32, so it differs
        from the dense call (TF32) by the TF32 rounding of the operator and the operands.

        `prune` (an extension): a list of (iter, keep) pairs with the rules of `rec_prune`, to prune restarts in this call:
        from iteration iter_k on each image runs only its keep_k restarts of lowest measured loss at iteration iter_k - 1
        (ties: the lower restart index; NaN last), and the arg-min picks among the last survivors (`return_aux`'s restart
        is the original index).  The survivors follow exactly their unpruned trajectories.  The schedule is checked
        before any native call (a ValueError naming the bad point) and refused with use_bn.  The measured call takes its
        schedule per call rather than from `rec_prune`, which is tuned for the image loss and names the reconstruction
        cache: without `prune`, a call with `rec_prune` set raises a ValueError; `prune=None` runs every restart to the
        end whatever `rec_prune` holds.

        `rec_optimizer`, `rec_adam_betas` and `rec_adam_eps` are read at call time as in `reconstruct`: with "adam" the
        measured loop updates z with Adam (rec_lr is then a step in z units), pruned or not.

        `rec_huber_delta` is read at call time as in `reconstruct`: a delta replaces the squared error of each measurement
        residual by the Huber loss, (1/m) sum_j rho(r_j), for a few corrupted measurements, dense or sparse, pruned or not.

        `operator` may also be a `defensegan_b200.operators.ConvOperator`: a blur, box downsample or blurred decimation,
        with one kernel for every image or one per image (deblurring photos with their own point-spread functions), applied
        as a stencil.  m is its num_measurements(image_dim); a per-image kernel count must equal B.  On both precisions
        the result is bit-identical to the call with its to_sparse_csr matrix (one call per image for per-image kernels),
        and it runs with prune, rec_optimizer and rec_huber_delta as the other operator kinds do.

        `rec_z_prior` is read at call time as in `reconstruct`: a lambda >= 0 adds lambda ||z||^2 to the measured loss,
        (1/m) ||A G(z) - y||^2 + lambda ||z||^2 - the latent prior of compressed sensing with generative models, with the
        data term normalised by m (the lambda of the unnormalised formulation is m times this one) - for every operator
        kind, pruned or not.

        `rec_sparse_dev` is read at call time as in `reconstruct`: each restart fits A (G(z) + nu) to y with an l1 penalty
        on the pixel-space deviation nu, whose step is step * m / 2 (step = 1 is the 1/Lipschitz step for ||A||_2 <= 1,
        such as the normalised blurs and box averages of ConvOperator), for every operator kind, pruned or not;
        `deviation_out` receives the chosen restart's nu."""
        adam = self._adam_params()
        huber = self._huber_delta()
        prior = self._z_prior()
        sdev = self._sparse_dev(deviation_out)
        if prune is _NOT_GIVEN:
            if self.rec_prune is not None:
                raise ValueError("rec_prune is set, but reconstruct_measured does not prune restarts from it: set "
                                 "rec_prune = None, or pass prune= to prune this call")
            prune = None
        if prune is not None:
            if bool(self.use_bn):
                raise ValueError("prune is not supported with use_bn: the batch statistics couple the restarts, so "
                                 "dropping some would change the others' trajectories")
            prune = _native.check_prune_schedule(prune, int(self.rec_rr), int(self.rec_iters))
        if isinstance(operator, ConvOperator):
            return self._reconstruct_measured_conv(measurements, operator, batch_size, z_init_val, return_aux, out,
                                                   z_row_offset, prune, adam, huber, prior, sdev, deviation_out)
        if isinstance(operator, torch.Tensor) and operator.layout in (torch.sparse_coo, torch.sparse_csr):
            return self._reconstruct_measured_sparse(measurements, operator, batch_size, z_init_val, return_aux, out,
                                                     z_row_offset, prune, adam, huber, prior, sdev, deviation_out)
        a = self._as_cuda(operator)
        hwc = int(np.prod(self.image_dim))
        if a.dim() != 2 or a.shape[1] != hwc or not 1 <= a.shape[0] <= hwc:
            raise ValueError("operator must be [m, %d] with 1 <= m <= %d (H*W*C), got %s" % (hwc, hwc, tuple(a.shape)))
        y = self._as_cuda(measurements).to(a.device)
        if y.dim() != 2 or y.shape[1] != a.shape[0] or y.shape[0] == 0:
            raise ValueError("measurements must be [B, %d] (one row of m values per image), got %s"
                             % (a.shape[0], tuple(y.shape)))
        if batch_size is not None and int(batch_size) != y.shape[0]:
            raise ValueError("batch_size (%d) does not match measurements.shape[0] (%d)" % (int(batch_size), y.shape[0]))
        finite = torch.stack([torch.isfinite(a).all(), torch.isfinite(y).all()]).tolist()
        bad = [name for name, ok in zip(("operator", "measurements"), finite) if not ok]
        if bad:
            raise ValueError("%s must be finite" % " and ".join(bad))
        z0 = self._as_cuda(z_init_val) if z_init_val is not None else None
        native = self._get_native(a.device)
        self.last_seed = seed = self._next_seed(0)
        kw = self._option_kwargs(adam, huber, prior, sdev, deviation_out)
        return native.reconstruct_measured(y, a, int(self.rec_rr), int(self.rec_iters), float(self.rec_lr), z_init_val=z0,
                                           seed=seed, momentum=float(self.rec_momentum), decay_lr=bool(self.rec_decay_lr),
                                           out=out, return_aux=return_aux, z_row_offset=int(z_row_offset), prune=prune,
                                           **kw)

    def _reconstruct_measured_conv(self, measurements, operator, batch_size, z_init_val, return_aux, out, z_row_offset,
                                   prune, adam=None, huber=None, prior=None, sdev=None, deviation_out=None):
        """reconstruct_measured for a ConvOperator, after one check of the kernels and the measurements (prune, adam,
        huber, prior, sdev and deviation_out as in _reconstruct_measured_sparse).  The native call gets the kernels broadcast to [B, kh, kw]."""
        m = operator.num_measurements(self.image_dim)
        y = self._as_cuda(measurements)
        if y.dim() != 2 or y.shape[1] != m or y.shape[0] == 0:
            raise ValueError("measurements must be [B, %d] (one row of the operator's m values per image), got %s"
                             % (m, tuple(y.shape)))
        b = y.shape[0]
        if batch_size is not None and int(batch_size) != b:
            raise ValueError("batch_size (%d) does not match measurements.shape[0] (%d)" % (int(batch_size), b))
        if operator.per_image and operator.kernel.shape[0] != b:
            raise ValueError("operator has %d per-image kernels for %d images (measurements.shape[0])"
                             % (operator.kernel.shape[0], b))
        k = operator.kernels(b, y.device)
        finite = torch.stack([torch.isfinite(k).all(), torch.isfinite(y).all()]).tolist()
        bad = [name for name, ok in zip(("operator kernels", "measurements"), finite) if not ok]
        if bad:
            raise ValueError("%s must be finite" % " and ".join(bad))
        z0 = self._as_cuda(z_init_val) if z_init_val is not None else None
        native = self._get_native(y.device)
        self.last_seed = seed = self._next_seed(0)
        kw = self._option_kwargs(adam, huber, prior, sdev, deviation_out)
        return native.reconstruct_measured(y, operator._with_kernels(k), int(self.rec_rr), int(self.rec_iters),
                                           float(self.rec_lr), z_init_val=z0, seed=seed,
                                           momentum=float(self.rec_momentum), decay_lr=bool(self.rec_decay_lr), out=out,
                                           return_aux=return_aux, z_row_offset=int(z_row_offset), prune=prune, **kw)

    def _reconstruct_measured_sparse(self, measurements, operator, batch_size, z_init_val, return_aux, out, z_row_offset,
                                     prune, adam=None, huber=None, prior=None, sdev=None, deviation_out=None):
        """reconstruct_measured for a sparse COO or CSR operator, after one check of the CSR and the measurements
        (prune: the checked schedule, or None; adam: the checked Adam parameters, or None; huber: the checked Huber delta,
        or None; prior: the checked latent prior's lambda, or None; sdev: the checked sparse deviations' (l1, step), or
        None, with deviation_out)."""
        a = operator
        if a.layout == torch.sparse_coo:
            if a.dim() != 2 or a.dense_dim() != 0:
                raise ValueError("operator must be a 2-D, non-hybrid sparse tensor, got %d dims (%d dense)"
                                 % (a.dim(), a.dense_dim()))
            a = a.coalesce().to_sparse_csr()
        if a.crow_indices().dim() != 1:
            raise ValueError("operator must not be a batched CSR tensor, got shape %s" % (tuple(a.shape),))
        if a.values().dim() != 1:
            raise ValueError("operator must not be a hybrid CSR tensor (values of shape %s)" % (tuple(a.values().shape),))
        hwc = int(np.prod(self.image_dim))
        if a.dim() != 2 or a.shape[1] != hwc or not 1 <= a.shape[0] <= hwc:
            raise ValueError("operator must be [m, %d] with 1 <= m <= %d (H*W*C), got %s" % (hwc, hwc, tuple(a.shape)))
        a = self._as_cuda(a)
        m = a.shape[0]
        y = self._as_cuda(measurements).to(a.device)
        if y.dim() != 2 or y.shape[1] != m or y.shape[0] == 0:
            raise ValueError("measurements must be [B, %d] (one row of m values per image), got %s" % (m, tuple(y.shape)))
        if batch_size is not None and int(batch_size) != y.shape[0]:
            raise ValueError("batch_size (%d) does not match measurements.shape[0] (%d)" % (int(batch_size), y.shape[0]))
        crow, col, val = a.crow_indices(), a.col_indices(), a.values()
        nnz = col.numel()
        # row starts: entry e + 1 opens a row when it is some row's first entry; otherwise its column must exceed e's
        start = torch.zeros(nnz + 1, dtype=torch.bool, device=col.device)
        start[crow.clamp(0, nnz)] = True
        checks = [
            ("operator crow_indices must rise from 0 to nnz = %d" % nnz,
             (crow[0] == 0) & (crow[-1] == nnz) & (crow[1:] >= crow[:-1]).all()),
            ("operator column indices must be in [0, %d)" % hwc, ((col >= 0) & (col < hwc)).all()),
            ("operator column indices must be strictly ascending within each row (no duplicates)",
             ((col[1:] > col[:-1]) | start[1:nnz]).all()),
            ("operator values must be finite", torch.isfinite(val).all()),
            ("measurements must be finite", torch.isfinite(y).all()),
        ]
        ok = torch.stack([c for _, c in checks]).tolist()
        bad = [name for (name, _), good in zip(checks, ok) if not good]
        if bad:
            raise ValueError("; ".join(bad))
        z0 = self._as_cuda(z_init_val) if z_init_val is not None else None
        native = self._get_native(a.device)
        self.last_seed = seed = self._next_seed(0)
        kw = self._option_kwargs(adam, huber, prior, sdev, deviation_out)
        return native.reconstruct_measured(y, a, int(self.rec_rr), int(self.rec_iters), float(self.rec_lr), z_init_val=z0,
                                           seed=seed, momentum=float(self.rec_momentum), decay_lr=bool(self.rec_decay_lr),
                                           out=out, return_aux=return_aux, z_row_offset=int(z_row_offset), prune=prune,
                                           **kw)

    def _pixel_weights(self, pixel_weights, x):
        """pixel_weights broadcast to x's shape and materialised once, after one check of all values (finite, in [0, 1])."""
        w = self._as_cuda(pixel_weights)
        try:
            w = torch.broadcast_to(w.to(x.device), x.shape).contiguous()
        except RuntimeError as e:
            raise ValueError("pixel_weights of shape %s do not broadcast to the images' shape %s"
                             % (tuple(w.shape), tuple(x.shape))) from e
        if not bool((torch.isfinite(w) & (w >= 0) & (w <= 1)).all()):
            raise ValueError("pixel_weights must be finite and in [0, 1]")
        return w

    # -- bulk offline reconstruction + its on-disk cache (reference models/gan.py:451-587, 604-646) --------------
    def set_dataset_generators(self, train: Optional[Callable] = None, dev: Optional[Callable] = None,
                               test: Optional[Callable] = None) -> None:
        """The reference binds `train_gen_test` / `dev_gen_test` / `test_gen_test` to its dataset readers
        (models/gan.py:666-673; out of scope here).  Each is a zero-argument callable returning an iterable of
        `(images, targets)` batches of RAW images (what `real_data_test_pl` is fed with); `input_transform` is applied."""
        if train is not None:
            self.train_gen_test = train
        if dev is not None:
            self.dev_gen_test = dev
        if test is not None:
            self.test_gen_test = test

    def rec_cache_dir(self, split: str, max_num: int = -1) -> str:
        """`<checkpoint_dir>/recs_rr{R}_lr{lr:.5f}_iters{L}[_num{n}][_prune{it}x{keep}[-{it}x{keep}...]]
        [_adam{b1:g}-{b2:g}-{eps:g}][_huber{delta:g}][_zprior{lambda:g}][_sdev{l1:g}_{step:g}]/<split>[_debug]` - the
        directory name the callers
        parse back with `recs_rr(.*)_lr(.*)_iters(.*)` (blackbox.py:646-651); the `_prune` part (only with `rec_prune` set)
        keeps pruned and unpruned reconstructions apart, the `_adam` part (only with rec_optimizer "adam") Adam's from
        momentum's, the `_huber` part (only with rec_huber_delta set) the Huber loss's from the squared error's, and the
        `_zprior` part (only with rec_z_prior set) those with the latent prior from those without, and the `_sdev` part
        (only with rec_sparse_dev set) those with sparse deviations from those without."""
        if max_num > 0:
            name = 'recs_rr{:d}_lr{:.5f}_iters{:d}_num{:d}'.format(int(self.rec_rr), float(self.rec_lr),
                                                                   int(self.rec_iters), int(max_num))
        else:
            name = 'recs_rr{:d}_lr{:.5f}_iters{:d}'.format(int(self.rec_rr), float(self.rec_lr), int(self.rec_iters))
        if self.rec_prune is not None:
            name += '_prune' + '-'.join('{:d}x{:d}'.format(int(it), int(keep)) for it, keep in self.rec_prune)
        adam = self._adam_params()
        if adam is not None:
            name += '_adam{:g}-{:g}-{:g}'.format(*adam)
        huber = self._huber_delta()
        if huber is not None:
            name += '_huber{:g}'.format(huber)
        prior = self._z_prior()
        if prior is not None:
            name += '_zprior{:g}'.format(prior)
        sdev = self._sparse_dev()
        if sdev is not None:
            name += '_sdev{:g}_{:g}'.format(*sdev)
        out = os.path.join(self.checkpoint_dir, name, split)
        if self.debug:
            out += '_debug'
        return out

    def _transformed_batch(self, images) -> torch.Tensor:
        x = self.input_transform(np.asarray(images))
        x = x.reshape([-1] + list(self.image_dim))
        return x

    def _dataset_projector(self):
        """(project, is_writer, agree) for reconstruct_dataset.  One process: `self.reconstruct`.  Under
        torch.distributed with several ranks (the bulk offline job on the 8 GPUs of a box): every rank walks the same
        batches, each batch is sharded over the ranks (`parallel.reconstruct_sharded`, one all-gather), rank 0 alone
        writes the cache and its hit / miss decisions are broadcast so that no rank can skip a collective another
        rank enters."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1):
            return self.reconstruct, True, (lambda flag: flag)
        from ..parallel import reconstruct_sharded
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu")

        def project(x):
            return reconstruct_sharded(self, x.to(dev))

        def agree(flag):
            t = torch.tensor([1 if flag else 0], dtype=torch.int32, device=dev)
            dist.broadcast(t, src=0)
            return bool(t.item())

        return project, dist.get_rank() == 0, agree

    def reconstruct_dataset(self, ckpt_path=None, max_num=-1, max_num_load=-1):
        """Projects the train/dev/test splits batch by batch (fresh z0 and zero momentum per batch, reference
        models/gan.py:541) behind the reference's two-level result cache (see `RecCache`).  Returns
        `{split: [all_recs, all_targets, orig_imgs]}` (numpy, images `[-1] + image_dim`), the reference's return value
        (models/gan.py:451-587).  Called on every rank of an initialised torch.distributed group it splits each batch
        over the ranks (`_dataset_projector`); every rank returns the full result."""
        if not self.initialized:
            self.load_generator(ckpt_path=ckpt_path)
        limit = max(max_num, max_num_load)
        shape = [-1] + list(self.image_dim)
        results = {}
        project, is_writer, agree = self._dataset_projector()
        for split in ('train', 'dev', 'test'):
            batches = getattr(self, split + '_gen_test', None)
            if batches is None:
                raise RuntimeError("no '{}_gen_test' generator bound: call set_dataset_generators(...) first "
                                   "(dataset readers are outside this package)".format(split))
            cache = RecCache(self.rec_cache_dir(split, max_num), reuse=not self.test_again)
            whole_split = cache.load_split()
            if not agree(whole_split is not None):          # rank 0's view of the cache decides for everybody
                whole_split = None
            elif whole_split is None:
                raise RuntimeError("rank 0 read {} but this rank cannot (the cache must be on a file system all "
                                   "ranks see)".format(cache.split_path))
            recs, targets, originals = [], [], []
            t_start = time.time()
            first = 0                                   # position of the batch's first image in the split
            for b, (images, labels) in enumerate(batches()):
                n = len(images)
                if (limit > -1 and first > limit) or (self.debug and b > 2):
                    break
                x = self._transformed_batch(images)
                if whole_split is None:
                    r = cache.load_batch(first, labels)
                    if not agree(r is not None):
                        r = project(x).detach().cpu().numpy()
                        if is_writer:
                            cache.store_batch(first, labels, r)
                            if self.verbose:
                                print('[rec] {} batch {:d}: projected in {:.2f} s'.format(split, b, time.time() - t_start))
                    elif r is None:
                        raise RuntimeError("rank 0 found batch {:d} of '{}' in {} but this rank cannot read it".format(
                            b, split, cache.pickle_dir))
                    recs.append(r)
                targets.append(np.asarray(labels))
                originals.append(np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x))
                first += n
            empty = np.zeros([0] + list(self.image_dim), dtype=np.float32)
            if whole_split is not None:
                all_recs = whole_split
            else:
                all_recs = np.concatenate(recs).reshape(shape) if recs else empty
            results[split] = [all_recs,
                              np.concatenate(targets) if targets else np.zeros([0], dtype=np.int64),
                              np.concatenate(originals).reshape(shape) if originals else empty]
        return results

    def save_recs(self, rets: Dict, max_num: int = -1) -> None:
        """Write each split's `feats.pkl` so that the next reconstruct_dataset (and the callers' cache loaders,
        blackbox.py:249-259,294-329) short-cut.  The reference leaves this to train.py --save_recs."""
        for split, (all_recs, _, _) in rets.items():
            RecCache(self.rec_cache_dir(split, max_num)).store_split(all_recs)

    def save_ds(self):
        """Dump the input-transformed dataset: `data/cache/<dataset>_pkl/<split>/feats.pkl` holding two
        consecutive pickles (images, targets) - the layout blackbox.get_cached_gan_data reads (:332-367)."""
        for split in ['train', 'dev', 'test']:
            output_dir = os.path.join('data', 'cache', '{}_pkl'.format(self.dataset_name), split)
            if self.debug:
                output_dir += '_debug'
            os.makedirs(output_dir, exist_ok=True)
            path = os.path.join(output_dir, 'feats.pkl')
            if os.path.exists(path) and not self.test_again:
                print('[#] Dataset is already saved.')
                return
            gen_func = getattr(self, '{}_gen_test'.format(split))
            imgs, tgts = [], []
            for images, targets in gen_func():
                x = self._transformed_batch(images)
                imgs.append(np.asarray(x.cpu() if isinstance(x, torch.Tensor) else x))
                tgts.append(np.asarray(targets))
            with open(path, 'wb') as f:
                pickle.dump(np.concatenate(imgs).reshape([-1] + list(self.image_dim)), f, pickle.HIGHEST_PROTOCOL)
                pickle.dump(np.concatenate(tgts), f, pickle.HIGHEST_PROTOCOL)

    def close(self):
        self._drop_native()


class MnistDefenseGAN(DefenseGANBase):
    """reference models/gan.py:649-685"""
    _dataset_default = "mnist"
    _image_dim_default = [28, 28, 1]

    def input_transform(self, X):
        return torch.as_tensor(X).to(torch.float32) / 255.0


class FmnistDefenseDefenseGAN(MnistDefenseGAN):
    """reference models/gan.py:688-698 (same generator as MNIST, different weights/data)"""
    _dataset_default = "f-mnist"


class CelebADefenseGAN(DefenseGANBase):
    """reference models/gan.py:718-765"""
    _dataset_default = "celeba"
    _image_dim_default = [64, 64, 3]

    def input_transform(self, images):
        return 2 * ((torch.as_tensor(images).to(torch.float32) / 255.0) - 0.5)

    def imsave_transform(self, imgs):
        imgs = (imgs + 1.0) / 2
        return imgs.clamp(0.0, 1.0) if isinstance(imgs, torch.Tensor) else np.clip(imgs, 0.0, 1.0)


# reference blackbox.py:56-61 / whitebox.py:49-53
dataset_gan_dict = {
    "mnist": MnistDefenseGAN,
    "f-mnist": FmnistDefenseDefenseGAN,
    "celeba": CelebADefenseGAN,
}
