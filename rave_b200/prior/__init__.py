"""The latent prior of rave/prior (scripts/train_prior.py): a WaveNet-style autoregressive model over the quantised PCA
latents of a pretrained, frozen RAVE.  `VariationalPrior.training_step` runs on the library's kernels (csrc/prior.cu and
the wgmma conv engine); see DESIGN.md §5.8."""
from .core import DiagonalShift, QuantizedNormal  # noqa: F401
from .model import GraphedPriorTrainer, Prior, VariationalPrior  # noqa: F401
from .residual_block import ResidualBlock  # noqa: F401
