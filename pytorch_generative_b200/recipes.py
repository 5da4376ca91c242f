"""`reproduce()` of the recipes — same signature, hyper-parameters, optimizer, scheduler, loss and data as reference
models/autoregressive/{pixel_cnn.py:113-176, gated_pixel_cnn.py:193-250, pixel_snail.py:190-262,
image_gpt.py:112-176, made.py:136-189, nade.py:93-146, fvbn.py:48-97}, models/flow/nice.py:164-226 and
models/vae/{vae.py:104-171, beta_vae.py:63-131, vq_vae.py:84-153, vq_vae_2.py:116-185, vd_vae.py:415-491}, on the CUDA path: the model classes of this package, the fused recipe losses, `FusedAdam` and this
package's `Trainer`.  Each model module re-exports its recipe as `reproduce`, like the reference's `train.py` expects.
"""

import torch

from . import losses, optim, trainer


def recipe_loss(x, _, preds):
    """loss_fn(x, _, preds) of every recipe: BCEWithLogits summed over the image, averaged over the batch."""
    return losses.bce_with_logits_sum_mean(preds, x)


def _run(model, lr, lr_gamma, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader, loss_fn=recipe_loss,
         transform=None, dataset="mnist"):
    """Trains `model` with FusedAdam on `dataset` ("mnist" or "cifar10"); `transform`: the loaders' data transform
    keywords (default for MNIST: dynamic binarisation)."""
    if n_gpus < 1:
        raise RuntimeError("the CUDA path trains on CUDA devices only (n_gpus >= 1); there is no CPU fallback")
    train_loader, test_loader = debug_loader, debug_loader
    if train_loader is None:
        from . import datasets

        device = torch.device("cuda", device_id or 0)
        if dataset == "cifar10":
            train_loader, test_loader = datasets.get_cifar10_loaders(batch_size, device=device, **(transform or {}))
        else:
            transform = transform or {"dynamically_binarize": True}
            train_loader, test_loader = datasets.get_mnist_loaders(batch_size, device=device, **transform)
    optimizer = optim.FusedAdam(model.parameters(), lr=lr)
    scheduler = None  # lr_gamma=None: a recipe without a learning-rate schedule
    if lr_gamma is not None:
        scheduler = torch.optim.lr_scheduler.MultiplicativeLR(optimizer, lr_lambda=lambda _: lr_gamma)
    model_trainer = trainer.Trainer(model=model, loss_fn=loss_fn, optimizer=optimizer, train_loader=train_loader,
                                    eval_loader=test_loader, lr_scheduler=scheduler, log_dir=log_dir, n_gpus=n_gpus,
                                    device_id=device_id)
    model_trainer.interleaved_train_and_eval(n_epochs)
    return model_trainer


def reproduce_pixel_cnn(n_epochs=457, batch_size=256, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.PixelCNN(in_channels=1, out_channels=1, n_residual=15, residual_channels=16, head_channels=32)
    return _run(model, 1e-3, 0.999977, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader)


def reproduce_gated_pixel_cnn(n_epochs=457, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.GatedPixelCNN(in_channels=1, out_channels=1, n_gated=10, gated_channels=128, head_channels=32)
    return _run(model, 1e-3, 0.9999, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader)


def reproduce_pixel_snail(n_epochs=457, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.PixelSNAIL(in_channels=1, out_channels=1, n_channels=64, n_pixel_snail_blocks=8, n_residual_blocks=2,
                              attention_value_channels=32, attention_key_channels=4)
    return _run(model, 1e-3, 0.999977, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader)


def reproduce_pixel_snail_8bit(n_epochs=457, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0,
                               debug_loader=None):
    """PixelSNAIL with `reproduce_pixel_snail`'s network, optimizer and schedule on CIFAR-10 scaled to [0, 1], with a
    discretised mixture of 10 logistics per pixel (`out_channels = 10 * 10`, `losses.logistic_mixture_nll`, which also
    logs bits/dim), the likelihood the PixelSNAIL paper reports CIFAR-10 bits/dim with.  The reference has no such
    recipe: convergence at these settings is not validated."""
    from . import models

    model = models.PixelSNAIL(in_channels=3, out_channels=100, n_channels=64, n_pixel_snail_blocks=8,
                              n_residual_blocks=2, attention_value_channels=32, attention_key_channels=4,
                              sample_fn=models.logistic_mixture_sample_fn(10, 256))
    return _run(model, 1e-3, 0.999977, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader,
                loss_fn=losses.logistic_mixture_nll, transform={"normalize": False}, dataset="cifar10")


def reproduce_image_gpt(n_epochs=457, batch_size=64, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.ImageGPT(in_channels=1, out_channels=1, in_size=28, n_transformer_blocks=8, n_attention_heads=2,
                            n_embedding_channels=64)
    return _run(model, 5e-3, 0.999977, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader)


def reproduce_image_gpt_8bit(n_epochs=457, batch_size=64, log_dir="/tmp/run", n_gpus=1, device_id=0,
                             debug_loader=None):
    """ImageGPT at the C5 shape of bench.py (24 blocks, 8 heads, 512 channels) on CIFAR-10 scaled to [0, 1], with a
    256-way categorical likelihood per sub-pixel (`out_channels = 256 * 3`, `losses.categorical_nll`, which also logs
    bits/dim) and `reproduce_image_gpt`'s optimizer and schedule.  The reference has no such recipe: convergence at
    these settings is not validated."""
    from . import models

    model = models.ImageGPT(in_channels=3, out_channels=256 * 3, in_size=32, n_transformer_blocks=24,
                            n_attention_heads=8, n_embedding_channels=512, sample_fn=models.categorical_sample_fn(256))
    return _run(model, 5e-3, 0.999977, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader,
                loss_fn=losses.categorical_nll, transform={"normalize": False}, dataset="cifar10")


def reproduce_made(n_epochs=85, batch_size=64, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.MADE(input_dim=784, hidden_dims=[8000], n_masks=1)
    return _run(model, 1e-3, None, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader)


def reproduce_nade(n_epochs=50, batch_size=512, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.NADE(input_dim=784, hidden_dim=500)
    return _run(model, 1e-3, None, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader)


def reproduce_fvbn(n_epochs=50, batch_size=512, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.FullyVisibleBeliefNetwork(n_dims=784)
    return _run(model, 1e-3, None, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader)


def reproduce_nice(n_epochs=150, batch_size=1024, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.NICE(n_features=784, n_coupling_blocks=4, n_hidden_layers=5, n_hidden_features=1000)
    return _run(model, 1e-3, None, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader,
                loss_fn=losses.logistic_prior_nll, transform={"dequantize": True})


def reproduce_vae(n_epochs=457, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.VAE(in_channels=1, out_channels=1, latent_channels=16, strides=[2, 2, 2, 2], hidden_channels=64,
                       residual_channels=32)
    return _run(model, 5e-4, None, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader,
                loss_fn=losses.vae_elbo, transform={"dynamically_binarize": True, "resize_to_32": True})


def reproduce_beta_vae(n_epochs=500, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.BetaVAE(in_channels=1, out_channels=1, beta=4.0, latent_channels=16, strides=[2, 2, 2, 2],
                           hidden_channels=64, residual_channels=32)
    return _run(model, 1e-3, None, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader,
                loss_fn=losses.vae_elbo, transform={"dynamically_binarize": True, "resize_to_32": True})


def reproduce_vq_vae(n_epochs=457, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.VectorQuantizedVAE(in_channels=3, out_channels=3, hidden_channels=128, residual_channels=32,
                                      n_residual_blocks=2, n_embeddings=512, embedding_dim=64)
    return _run(model, 2e-4, 0.999977, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader,
                loss_fn=losses.vq_vae_loss, transform={"normalize": True}, dataset="cifar10")


def reproduce_vq_vae_2(n_epochs=457, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models

    model = models.VectorQuantizedVAE2(in_channels=3, out_channels=3, hidden_channels=128, n_residual_blocks=2,
                                       residual_channels=64, n_embeddings=512, embedding_dim=64)
    return _run(model, 2e-4, 0.999977, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader,
                loss_fn=losses.vq_vae_2_loss, transform={"normalize": True}, dataset="cifar10")


def reproduce_vd_vae(n_epochs=500, batch_size=128, log_dir="/tmp/run", n_gpus=1, device_id=0, debug_loader=None):
    from . import models
    from .models.vd_vae import StackConfig

    stack_configs = [StackConfig(n_encoder_blocks=3, n_decoder_blocks=5), StackConfig(n_encoder_blocks=3, n_decoder_blocks=5),
                     StackConfig(n_encoder_blocks=2, n_decoder_blocks=4), StackConfig(n_encoder_blocks=2, n_decoder_blocks=3),
                     StackConfig(n_encoder_blocks=2, n_decoder_blocks=2), StackConfig(n_encoder_blocks=1, n_decoder_blocks=1)]
    model = models.VeryDeepVAE(in_channels=1, out_channels=1, input_resolution=32, stack_configs=stack_configs,
                               latent_channels=16, hidden_channels=64, bottleneck_channels=32)
    return _run(model, 5e-4, None, n_epochs, batch_size, log_dir, n_gpus, device_id, debug_loader,
                loss_fn=losses.vae_elbo, transform={"dynamically_binarize": True, "resize_to_32": True})
