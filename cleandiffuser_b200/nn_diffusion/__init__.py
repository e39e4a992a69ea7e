from .base import BaseNNDiffusion
from .unets import JannerUNet1d, ChiUNet1d, ResidualBlock, ChiResidualBlock, Downsample1d, Upsample1d
from .dit1d import DiT1d, DiTBlock, FinalLayer1d
from .chitransformer import ChiTransformer
from .mlp_dql import DQLMlp
from .mlp_idql import IDQLMlp
from .mlp_misc import DVInvMlp, SfBCUNet, PearceMlp
