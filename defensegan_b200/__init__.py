"""defensegan_b200 - H100-native (sm_90a) Defense-GAN projection loop behind the reference's Python surface.

Public surface (mirrors kabkabm/defensegan):
    defensegan_b200.models.gan.{MnistDefenseGAN, FmnistDefenseDefenseGAN, CelebADefenseGAN}
    defensegan_b200.utils.gan_defense.model_eval_gan
    defensegan_b200.utils.config.load_config
    defensegan_b200.utils.network_builder.{ReconstructionLayer, model_a ... model_z}
    defensegan_b200.blackbox.blackbox / defensegan_b200.whitebox.whitebox   (the experiment drivers; also `python -m`)
    defensegan_b200.train   (`--save_recs` / `--save_ds`: the caches those drivers read)
    defensegan_b200.parallel.reconstruct_sharded   (image axis over the GPUs of a box, one all-gather)
Native layer: defensegan_b200._native (ctypes over include/defensegan_b200.h).
"""
__version__ = "0.1.0"
