"""What the attack scripts (blackbox.py / whitebox.py) share: flags, cached-dataset access, result files.

The reference keeps these as module-level `tf.app.flags` and copies of the same helper code in both scripts
(blackbox.py:216-367,596-700, whitebox.py:239-342).  Here the flags are one plain object passed around, the cached
data comes back as a `SplitData`, and the result-file logic is a function of (flags, gan).

Datasets themselves (MNIST / F-MNIST / CelebA readers) are outside this package: the scripts consume the on-disk
caches that `DefenseGANBase.save_ds` (original images) and `reconstruct_dataset` / `save_recs` (reconstructions) write,
or arrays handed in directly.
"""
from __future__ import annotations

import argparse
import collections
import os
import pickle
import re
from typing import Optional

import numpy as np

SplitData = collections.namedtuple("SplitData", "train_images train_labels test_images test_labels")

# flag -> (type, default): the union of the two scripts' `flags.DEFINE_*` lists (blackbox.py:723-759,
# whitebox.py:362-392; where they differ the script's own default is applied by `script_defaults`)
_FLAG_TABLE = collections.OrderedDict([
    ("nb_classes", (int, 10)), ("learning_rate", (float, 0.001)), ("nb_epochs", (int, 10)), ("holdout", (int, 150)),
    ("data_aug", (int, 6)), ("nb_epochs_s", (int, 10)), ("lmbda", (float, 0.1)), ("fgsm_eps", (float, 0.3)),
    ("fgsm_eps_tr", (float, 0.15)), ("rec_path", (str, None)), ("num_tests", (int, -1)), ("random_test_iter", (int, -1)),
    ("online_training", (bool, False)), ("defense_type", (str, "none")), ("attack_type", (str, "none")),
    ("results_dir", (str, None)), ("train_on_recs", (bool, False)), ("num_train", (int, -1)), ("bb_model", (str, "F")),
    ("sub_model", (str, "E")), ("model", (str, "F")), ("same_init", (bool, False)), ("debug_dir", (str, None)),
    ("debug", (bool, False)), ("override", (bool, False)), ("alpha", (float, 0.05)), ("test_on_dev", (bool, True)),
])
script_defaults = {"blackbox": {"num_tests": 2000}, "whitebox": {"num_tests": -1, "debug_dir": "temp"}}


def _flag_bool(v):
    if isinstance(v, bool):
        return v
    s = str(v).lower()
    if s in ("true", "t", "1", "yes", "y"):
        return True
    if s in ("false", "f", "0", "no", "n"):
        return False
    raise argparse.ArgumentTypeError("boolean value expected, got %r" % (v,))


class Flags(argparse.Namespace):
    """The scripts' flag values as attributes.  Unknown names read as None (like an undefined optional flag), so the
    same object serves both scripts."""

    def __init__(self, script: Optional[str] = None, **values):
        super().__init__()
        for name, (_, default) in _FLAG_TABLE.items():
            setattr(self, name, default)
        for name, default in script_defaults.get(script or "", {}).items():
            setattr(self, name, default)
        for name, v in values.items():
            setattr(self, name, v)

    def __getattr__(self, name):          # only reached for attributes that were never set
        if name.startswith("__"):
            raise AttributeError(name)
        return None


def add_script_flags(parser: argparse.ArgumentParser, script: str) -> argparse.ArgumentParser:
    """`--<flag>` options of one script on top of the cfg-derived ones (`utils.config.add_flags`)."""
    defaults = dict((k, d) for k, (_, d) in _FLAG_TABLE.items())
    defaults.update(script_defaults.get(script, {}))
    for name, (typ, _) in _FLAG_TABLE.items():
        opt = "--" + name
        if any(opt in a.option_strings for a in parser._actions):
            continue
        parser.add_argument(opt, type=_flag_bool if typ is bool else typ, default=defaults[name])
    return parser


def convert_to_onehot(ys) -> np.ndarray:
    """Integer labels -> float32 one-hot rows, max(label) + 1 columns (blackbox.py:216-222)."""
    ys = np.asarray(ys).astype(np.int64).ravel()
    out = np.zeros((len(ys), int(ys.max()) + 1 if len(ys) else 0), np.float32)
    out[np.arange(len(ys)), ys] = 1.0
    return out


# ------------------------------------------------------------------------------------------------------------------
# cached datasets
# ------------------------------------------------------------------------------------------------------------------
def orig_data_path(dataset_name: str) -> str:
    """Where `save_ds` puts the input-transformed dataset (blackbox.py:61-62)."""
    return os.path.join("data", "cache", "{}_pkl".format(dataset_name))


def _load_feats(path):
    """`feats.pkl` as save_ds writes it: two consecutive pickles (images, integer targets)."""
    with open(path, "rb") as f:
        return pickle.load(f), pickle.load(f)


def get_train_test(data_path, test_on_dev=True, model=None, orig_data=False, max_num=-1) -> SplitData:
    """Train + evaluation split for the classifier (blackbox.py:272-329).  `orig_data=True`: the cached original images
    under `data_path`.  Otherwise `model.reconstruct_dataset(max_num_load=max_num)` supplies reconstructions (and the
    originals).  This is the documented contract of the reference's function (:277-282); as written the reference
    returns the cached ORIGINALS whenever `feats.pkl` loads, even for `orig_data=False` (:300-321, the reconstructions
    are only a fall-back for an unreadable cache) - that quirk is not reproduced.
    The reference's split naming is kept: `test_on_dev=True` selects the split called 'test', False 'dev' (:323)."""
    rec_sets = model.reconstruct_dataset(max_num_load=max_num) if (model is not None and not orig_data) else None
    out = []
    for split in ("train", "test" if test_on_dev else "dev"):
        feats = os.path.join(data_path, split, "feats.pkl")
        images = labels = None
        if rec_sets is None or orig_data:
            if not os.path.exists(feats):
                raise IOError("{} is missing: dump the dataset cache first (gan.save_ds(); the reference's "
                              "`python train.py --cfg <cfg> --save_ds`)".format(feats))
            try:
                images, labels = _load_feats(feats)
            except Exception as e:                      # unreadable cache: fall through to the live reconstructions
                print("[!] Found feats.pkl but could not load it because {}".format(e))
        if images is None:
            if rec_sets is None:
                raise IOError("no usable data for split '{}' under {}".format(split, data_path))
            recs, labels, originals = rec_sets[split]
            images = originals if orig_data else recs
        out += [np.asarray(images), convert_to_onehot(labels)]
    return SplitData(*out)


def get_pickle_split(rec_path, split, image_dim):
    """One split of a reconstruction cache read image by image: `<rec_path>/<split>/pickles/rec_{i:07d}_l{label}.pkl`
    (what the reference's CelebA branch does lazily, blackbox.py:249-259).  Returns (images, integer labels) in index
    order - the label is parsed from the file name."""
    d = os.path.join(rec_path, split, "pickles")
    if not os.path.isdir(d):
        raise IOError("no reconstruction pickles at {}".format(d))
    names = sorted(n for n in os.listdir(d) if re.match(r".*_l(\d+)\.pkl$", n))
    labels = np.array([int(re.match(r".*_l(\d+)\.pkl$", n).group(1)) for n in names], np.int32)
    images = np.zeros([len(names)] + list(image_dim), np.float32)
    for i, n in enumerate(names):
        with open(os.path.join(d, n), "rb") as f:
            images[i] = np.asarray(pickle.load(f)).reshape(image_dim)
    return images, labels


def get_cached_gan_data(gan, test_on_dev, orig_data_flag=None, flags: Optional[Flags] = None) -> SplitData:
    """The data a script trains / evaluates on (blackbox.py:332-367).  `orig_data_flag=None`: originals unless the
    classifier is to be trained on Defense-GAN reconstructions (`--train_on_recs` with `--defense_type defense_gan`)."""
    flags = flags if flags is not None else Flags()
    if orig_data_flag is None:
        orig_data_flag = not (flags.train_on_recs and flags.defense_type == "defense_gan")
    if "celeba" in str(gan.dataset_name) and not orig_data_flag:
        # CelebA reconstructions are consumed from the per-image pickles of --rec_path (blackbox.py:225-269)
        dev = "val" if test_on_dev else "test"
        tr_x, tr_y = get_pickle_split(flags.rec_path, "train", gan.image_dim)
        te_x, te_y = get_pickle_split(flags.rec_path, dev, gan.image_dim)
        data = SplitData(tr_x, convert_to_onehot(tr_y), te_x, convert_to_onehot(te_y))
    else:
        data = get_train_test(orig_data_path(gan.dataset_name), test_on_dev=test_on_dev, model=gan,
                              orig_data=orig_data_flag, max_num=flags.num_train)
    if "celeba" in str(gan.dataset_name) and flags.num_train and flags.num_train > 0:
        data = data._replace(train_images=data.train_images[:flags.num_train],
                             train_labels=data.train_labels[:flags.num_train])
    return data


# ------------------------------------------------------------------------------------------------------------------
# reconstruction hyper-parameters and result files
# ------------------------------------------------------------------------------------------------------------------
_REC_DIR_RE = re.compile(r"recs_rr(.*)_lr(.*)_iters(.*)")
_REC_PRUNE_RE = re.compile(r"_prune(\d+x\d+(?:-\d+x\d+)*)")
_G = r"(\d+(?:\.\d*)?(?:e[-+]\d+)?)"            # a number as '{:g}' writes it
_REC_ADAM_RE = re.compile(r"_adam%s-%s-%s" % (_G, _G, _G))
_REC_HUBER_RE = re.compile(r"_huber(inf|\d+(?:\.\d*)?(?:e[-+]\d+)?)")
_REC_ZPRIOR_RE = re.compile(r"_zprior%s" % _G)
_REC_SDEV_RE = re.compile(r"_sdev%s_%s" % (_G, _G))


def set_test_time_rec_params(gan, flags: Flags, cfg=None) -> None:
    """blackbox.py:639-658 / whitebox.py:245-264: with `--rec_path` and `--defense_type defense_gan` the projection's
    hyper-parameters are parsed back from the cache directory name (`rec_cache_dir`), the restart-pruning schedule
    (`_prune<it>x<keep>[-<it>x<keep>...]`) included: `gan.rec_prune` becomes that schedule, or None when the name has
    none; so is the optimiser (`_adam<b1>-<b2>-<eps>`): "adam" with those betas and eps, or "momentum" when the name
    has none; and the data term (`_huber<delta>`): the Huber loss at that delta, or the squared error (None) when the name
    has none; and the latent prior (`_zprior<lambda>`): that lambda, or no prior (None) when the name has none; and the
    sparse deviations (`_sdev<l1>_<step>`): that (l1, step), or none (None) when the name has none;
    `--override` applies the `--rec_rr / --rec_lr / --rec_iters` values instead of the model cfg's."""
    cfg = cfg or {}
    rr = cfg.get("REC_RR", gan.rec_rr)
    lr = cfg.get("REC_LR", gan.rec_lr)
    iters = cfg.get("REC_ITERS", gan.rec_iters)
    defense = str(flags.defense_type).lower()
    if defense != "none":
        if flags.rec_path and defense == "defense_gan":
            found = _REC_DIR_RE.findall(flags.rec_path)
            if not found:
                raise ValueError("--rec_path %r does not contain recs_rr<R>_lr<lr>_iters<L>" % (flags.rec_path,))
            rr, lr, iters = found[0]
            iters = re.split(r"[/_]", str(iters))[0]            # `..._iters200/train`, `..._iters200_num500`
            gan.rec_rr, gan.rec_lr, gan.rec_iters = int(rr), float(lr), int(iters)
            prune = _REC_PRUNE_RE.findall(flags.rec_path)
            gan.rec_prune = [tuple(int(v) for v in p.split("x")) for p in prune[0].split("-")] if prune else None
            adam = _REC_ADAM_RE.findall(flags.rec_path)
            if adam:
                b1, b2, eps = (float(v) for v in adam[0])
                gan.rec_optimizer, gan.rec_adam_betas, gan.rec_adam_eps = "adam", (b1, b2), eps
            else:
                gan.rec_optimizer = "momentum"
            huber = _REC_HUBER_RE.search(flags.rec_path)
            gan.rec_huber_delta = float(huber.group(1)) if huber else None
            prior = _REC_ZPRIOR_RE.search(flags.rec_path)
            gan.rec_z_prior = float(prior.group(1)) if prior else None
            sdev = _REC_SDEV_RE.search(flags.rec_path)
            gan.rec_sparse_dev = (float(sdev.group(1)), float(sdev.group(2))) if sdev else None
        elif defense == "defense_gan":
            assert flags.online_training or not flags.train_on_recs
    if flags.override:
        gan.rec_rr, gan.rec_lr, gan.rec_iters = int(rr), float(lr), int(iters)


def unique_result_path(results_dir, file_name):
    """`<results_dir>/<k>_<file_name>` with the smallest k that does not exist yet (blackbox.py:663-673)."""
    k = 0
    while os.path.exists(os.path.join(results_dir, "{}_{}".format(k, file_name))):
        k += 1
    return os.path.join(results_dir, "{}_{}".format(k, file_name))


def write_results(path, values, roc_info=None):
    """One line of space-separated values appended to `path`; `roc_info` ([labels, preds, diffs], for attack
    detection) goes to `<path minus .txt>_roc.pkl` (blackbox.py:687-699)."""
    os.makedirs(os.path.dirname(path) or ".", exist_ok=True)
    with open(path, "a") as f:
        f.write("".join(str(v) + " " for v in values) + "\n")
    print("[*] saved accuracy in {}".format(path))
    if roc_info:
        roc_path = path.replace(".txt", "_roc.pkl")
        with open(roc_path, "wb") as f:
            pickle.dump(roc_info, f, pickle.HIGHEST_PROTOCOL)
        print("[*] saved roc_info in {}".format(roc_path))
