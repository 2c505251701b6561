"""Default hot-path options of the reference as an ``argparse.Namespace`` (the reference assembles them from
every layer's ``modify_commandline_options``: options/__init__.py:30-51, swapping_autoencoder_model.py:12-23,
encoder.py:34-37, generator.py:95-102, discriminator.py:8, patch_discriminator.py:14-19,
swapping_autoencoder_optimizer.py:14-21).  bench.py and the tests build their configuration from here."""
from argparse import Namespace


def default_options(**overrides):
    opt = Namespace(
        # experiment / runtime
        name="sae_b200", checkpoints_dir="./checkpoints", isTrain=True, continue_train=False, pretrained_name=None,
        resume_iter="latest", num_gpus=1, batch_size=16, crop_size=256, load_size=256,
        # network selection
        model="swapping_autoencoder", optimizer="swapping_autoencoder",
        netE="StyleGAN2Resnet", netG="StyleGAN2Resnet", netD="StyleGAN2", netPatchD="StyleGAN2",
        use_antialias=True, num_classes=0,
        # loss graph
        spatial_code_ch=8, global_code_ch=2048, lambda_R1=10.0, lambda_patch_R1=1.0, lambda_L1=1.0, lambda_GAN=1.0,
        lambda_PatchGAN=1.0, patch_min_scale=1 / 8, patch_max_scale=1 / 4, patch_num_crops=8,
        patch_use_aggregation=True,
        # encoder
        netE_scale_capacity=1.0, netE_num_downsampling_sp=4, netE_num_downsampling_gl=2, netE_nc_steepness=2.0,
        # generator
        netG_scale_capacity=1.0, netG_num_base_resnet_layers=2, netG_use_noise=True, netG_resnet_ch=256,
        # discriminators
        netD_scale_capacity=1.0, netPatchD_scale_capacity=4.0, netPatchD_max_nc=256 + 128, patch_size=128,
        max_num_tiles=8, patch_random_transformation=False,
        # optimisation
        lr=0.002, beta1=0.0, beta2=0.99, R1_once_every=16,
        # extension (not a reference option): replay each half-step as a CUDA graph (graphs.py)
        cuda_graphs=False,
        # extension: run D (and Dpatch in the discriminator step) once over the concatenated real / rec / mix batch — per-sample
        # identical losses and gradients (tests/test_host_logic.py, 1e-10), same random draws in the same order, a third of the
        # discriminator launches and fuller tiles on the small late layers (+2.9 % images/s measured).  False: three passes,
        # literally as reference models/swapping_autoencoder_model.py:62-98 writes them.
        batch_discriminator_passes=True,
        # extension: losses are read back with one asynchronous copy per half-step and the host only waits when a value is
        # looked at (util.LazyLosses); False: the reference's blocking to_numpy
        async_loss_readback=True,
        # extension: scan the gradients of every half-step on the device and drop its Adam update when one of them holds a NaN
        # or an Inf (parameters, moments and step counts stay bitwise unchanged); nonfinite_steps() / nonfinite_report() tell
        # how often and where (optimizer.NonfiniteGuard)
        skip_nonfinite_steps=False,
        # extension: gradient accumulation — each rank's batch is split into this many micro-batches, run one after the other,
        # and one Adam update is made from their summed gradients, so the global batch no longer has to fit one pass per GPU
        # (SwappingAutoencoderOptimizer.split_micro_batches; INTEGRATION.md §2e)
        micro_batches=1,
        # extension: weight averaging — after every G update an exponential moving average of the E and G weights moves towards
        # them, with this half-life in thousands of images (0: off) and StyleGAN2-ADA's ramp-up (the half-life is at most
        # ema_rampup times the images seen so far; 0: no ramp); trainer.save writes it as <N>k_ema_checkpoint.pth
        # (optimizer.ParameterEMA; INTEGRATION.md §2f)
        ema_kimg=0.0, ema_rampup=0.05,
        # extension: training statistics — per-update gradient, weight and Adam-step norms of every group and the mean score and
        # sign of every discriminator logit tensor, accumulated on the device until trainer.training_stats() reads them
        # (optimizer.TrainingStats; INTEGRATION.md §2g)
        training_stats=False,
        # extension: adaptive discriminator augmentation — StyleGAN2-ADA's geometric and colour transforms of every input of D
        # with probability augment_p; ada_target > 0 tunes it on the device towards E[sign(D(real))] = ada_target, moving it
        # by up to one unit per ada_kimg thousand images, every ada_interval D updates; on iff augment_p > 0 or ada_target > 0
        # (augment.AugmentPipe; INTEGRATION.md §2h)
        augment_p=0.0, ada_target=0.0, ada_kimg=500.0, ada_interval=4,
    )
    for k, v in overrides.items():
        setattr(opt, k, v)
    return opt
