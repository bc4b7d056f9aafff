"""makani_b200 -- H100-native (sm_90a) implementation of makani's spherical-harmonic hot path.

Public surface (mirrors the reference, see INTEGRATION.md):
    RealSHT, InverseRealSHT                    <- torch_harmonics.{RealSHT, InverseRealSHT}
    RealVectorSHT, InverseRealVectorSHT        <- torch_harmonics.{RealVectorSHT, InverseRealVectorSHT} (makani's vort/div and gradient losses)
    DiscreteContinuousConvS2                   <- torch_harmonics.DiscreteContinuousConvS2 (FCN3's encoders, decoders and local blocks; morlet basis)
    DiscreteContinuousConvTransposeS2          <- torch_harmonics.DiscreteContinuousConvTransposeS2 (learnable upsampling; morlet basis)
    ResampleS2                                 <- torch_harmonics.ResampleS2 (FCN3's and SNO's decoders; mode "bilinear")
    NeighborhoodAttentionS2                    <- torch_harmonics.NeighborhoodAttentionS2 (local attention on the DISCO neighbourhoods)
    AttentionS2                                <- torch_harmonics.AttentionS2 (global attention, quadrature-weighted keys)
    SpectralConv, SpectralAttention, ComplexReLU <- makani.models.common.*
    quadrature                                 <- torch_harmonics.quadrature
    distributed                                <- torch_harmonics.distributed (h x w spatial model parallelism; its
                                                  DistributedNeighborhoodAttentionS2 and DistributedAttentionS2 are
                                                  NeighborhoodAttentionS2 and AttentionS2 on a sharded grid)
    install_torch_harmonics_shim()             <- makes `import torch_harmonics` resolve to this package
    HostFeed                                   <- double-buffered host->device input staging (the data loader's prefetch queue)
    sfno.SphericalFourierNeuralOperatorNet     <- makani.models.networks.sfnonet (same constructor / parameters / state dict)
    fcn3.AtmoSphericNeuralOperatorNet          <- makani.models.networks.fourcastnet3 (FourCastNet 3; same constructor / parameters / state dict;
                                                  also its NeuralOperatorBlock, DiscreteContinuousEncoder / Decoder, LayerScale); on
                                                  a grid set by distributed.init it builds makani's distributed modules and tags
    distributed.scatter_state_dict, gather_state_dict, sync_shared_params, reduce_shared_gradients
                                               <- makani.utils.checkpoint_helpers / mpu.helpers / the DDP comm hook of mpu.mappings
                                                  (global checkpoints and shared-parameter gradients under h x w)
    noise.DiffusionNoiseS2, noise.IsotropicGaussianRandomFieldS2, noise.DummyNoiseS2, noise.build_noise
                                               <- makani.models.noise (FCN3's input noise: the state update and the synthesis input on sm_90a)
    norm.InstanceNorm2d, norm.bias_gelu        <- torch.nn.InstanceNorm2d (+ GELU), bias + GELU on the library's kernels (row N2)
"""
from ._lib import B200ShtError, load as load_library  # noqa: F401
from . import quadrature  # noqa: F401
from .sht import RealSHT, InverseRealSHT, get_plan, resolve_precision  # noqa: F401
from .vector_sht import RealVectorSHT, InverseRealVectorSHT  # noqa: F401
from .disco import DiscreteContinuousConvS2, DiscreteContinuousConvTransposeS2  # noqa: F401
from .resample import ResampleS2  # noqa: F401
from .attention import NeighborhoodAttentionS2, AttentionS2  # noqa: F401
from .spectral_convolution import SpectralConv, SpectralAttention, ComplexReLU, mix_packed  # noqa: F401
from .host_pipeline import HostFeed  # noqa: F401
from . import noise  # noqa: F401

__version__ = "0.1.0"
