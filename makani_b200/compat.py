"""`torch_harmonics` shim: lets makani's own Python (networks, trainers, configs) run unchanged on top of makani_b200.

makani imports the package by name at module import time (`import torch_harmonics as th`,
`import torch_harmonics.distributed as thd`, `from torch_harmonics.distributed.primitives import ...`:
/root/reference/makani/models/networks/sfnonet.py:31-32, models/common/spectral_convolution.py:34, mpu/mappings.py:19-25)
and checks class identity (`isinstance(..., thd.DistributedInverseRealSHT)`, spectral_convolution.py:169), so the shim must be
registered in `sys.modules` BEFORE `import makani`:

    import makani_b200.compat as compat
    compat.install_torch_harmonics_shim()      # torch_harmonics -> makani_b200
    compat.patch_makani_spectral_layers()      # makani.models.common.SpectralConv/SpectralAttention -> makani_b200 (optional)
    compat.patch_makani_norm_layers()          # makani's (Distributed)GeometricInstanceNormS2 -> makani_b200 (optional)
    compat.patch_makani_layer_norm()           # makani's DistributedLayerNorm -> makani_b200 (optional)
    compat.patch_makani_instance_norm()        # makani's DistributedInstanceNorm2d -> makani_b200 (optional)
    import makani
"""
import importlib
import sys
import types


def install_torch_harmonics_shim(force=False):
    """Register `torch_harmonics`, `.quadrature`, `.filter_basis`, `.distributed`, `.distributed.primitives` backed by makani_b200."""
    if "torch_harmonics" in sys.modules and not force:
        mod = sys.modules["torch_harmonics"]
        if getattr(mod, "__b200_shim__", False):
            return mod
        raise RuntimeError("a real torch_harmonics is already imported; pass force=True to replace it")
    import makani_b200 as mb
    from makani_b200 import disco as mbdisco
    from makani_b200 import distributed as mbd   # with the distributed DISCO convolutions and DistributedResampleS2
    from makani_b200 import quadrature as mbq

    th = types.ModuleType("torch_harmonics")
    th.__b200_shim__ = True
    th.__version__ = "0.9.0+b200"
    th.RealSHT = mb.RealSHT
    th.InverseRealSHT = mb.InverseRealSHT
    th.RealVectorSHT = mb.RealVectorSHT
    th.InverseRealVectorSHT = mb.InverseRealVectorSHT
    th.DiscreteContinuousConvS2 = mb.DiscreteContinuousConvS2
    th.DiscreteContinuousConvTransposeS2 = mb.DiscreteContinuousConvTransposeS2
    th.ResampleS2 = mb.ResampleS2
    th.NeighborhoodAttentionS2 = mb.NeighborhoodAttentionS2
    th.AttentionS2 = mb.AttentionS2
    fb = types.ModuleType("torch_harmonics.filter_basis")
    fb.get_filter_basis, fb.MorletFilterBasis = mbdisco.get_filter_basis, mbdisco.MorletFilterBasis
    th.filter_basis = fb
    th.quadrature = mbq
    th.distributed = mbd
    th.__path__ = []  # mark as package so that submodule imports resolve through sys.modules
    sys.modules["torch_harmonics"] = th
    sys.modules["torch_harmonics.quadrature"] = mbq
    sys.modules["torch_harmonics.filter_basis"] = fb
    sys.modules["torch_harmonics.distributed"] = mbd
    sys.modules["torch_harmonics.distributed.primitives"] = mbd.primitives
    sys.modules["torch_harmonics.distributed.utils"] = mbd
    return th


def patch_makani_spectral_layers():
    """After `import makani`: point makani.models.common.{SpectralConv, SpectralAttention, ComplexReLU} at the CUDA-backed classes."""
    import makani_b200 as mb

    common = importlib.import_module("makani.models.common")
    for name in ("SpectralConv", "SpectralAttention", "ComplexReLU"):
        setattr(common, name, getattr(mb, name))
    sc = sys.modules.get("makani.models.common.spectral_convolution")
    if sc is not None:
        sc.SpectralConv = mb.SpectralConv
        sc.SpectralAttention = mb.SpectralAttention
    for modname in ("makani.models.networks.sfnonet", "makani.models.networks.fourcastnet3", "makani.models.networks.fourcastnet3_1", "makani.models.networks.snonet"):
        m = sys.modules.get(modname)
        if m is not None:
            for name in ("SpectralConv", "SpectralAttention"):
                if hasattr(m, name):
                    setattr(m, name, getattr(mb, name))


def patch_makani_norm_layers():
    """After `import makani`: point makani's GeometricInstanceNormS2 (makani.models.common, .layer_norm) and DistributedGeometricInstanceNormS2
    (makani.mpu.layer_norm) at the CUDA-backed classes, including the names the networks imported at module load."""
    from makani_b200 import distributed as mbd
    from makani_b200.norm import GeometricInstanceNormS2

    common = importlib.import_module("makani.models.common")
    common.GeometricInstanceNormS2 = GeometricInstanceNormS2
    for modname, name, cls in (("makani.models.common.layer_norm", "GeometricInstanceNormS2", GeometricInstanceNormS2),
                               ("makani.mpu.layer_norm", "DistributedGeometricInstanceNormS2", mbd.DistributedGeometricInstanceNormS2)):
        m = sys.modules.get(modname) or importlib.import_module(modname)
        setattr(m, name, cls)
    for modname in ("makani.models.networks.sfnonet", "makani.models.networks.snonet", "makani.models.networks.fourcastnet3",
                    "makani.models.networks.fourcastnet3_1"):
        m = sys.modules.get(modname)
        if m is not None:
            for name, cls in (("GeometricInstanceNormS2", GeometricInstanceNormS2), ("DistributedGeometricInstanceNormS2", mbd.DistributedGeometricInstanceNormS2)):
                if hasattr(m, name):
                    setattr(m, name, cls)


def patch_makani_layer_norm():
    """After `import makani`: point makani.mpu.layer_norm.DistributedLayerNorm at the CUDA-backed class, and the name that sfnonet / snonet imported
    at module load.  FourCastNet 3 and 3.1 import it inside a function, so the module attribute covers them.  makani's check that the matmul group
    has one rank stays in makani's own class; this library has no matmul group."""
    from makani_b200.norm import DistributedLayerNorm

    m = sys.modules.get("makani.mpu.layer_norm") or importlib.import_module("makani.mpu.layer_norm")
    m.DistributedLayerNorm = DistributedLayerNorm
    for modname in ("makani.models.networks.sfnonet", "makani.models.networks.snonet"):
        net = sys.modules.get(modname)
        if net is not None and hasattr(net, "DistributedLayerNorm"):
            net.DistributedLayerNorm = DistributedLayerNorm


def patch_makani_instance_norm():
    """After `import makani`: point makani.mpu.layer_norm.DistributedInstanceNorm2d (SFNO's default `instance_norm` when the spatial group has more
    than one rank) at the CUDA-backed class, and the name that sfnonet / snonet imported at module load.  FourCastNet 3 and 3.1 import it inside a
    function, so the module attribute covers them.  makani's DistributedGeometricInstanceNormS2 keeps its own base class."""
    from makani_b200.distributed import DistributedInstanceNorm2d

    m = sys.modules.get("makani.mpu.layer_norm") or importlib.import_module("makani.mpu.layer_norm")
    m.DistributedInstanceNorm2d = DistributedInstanceNorm2d
    for modname in ("makani.models.networks.sfnonet", "makani.models.networks.snonet"):
        net = sys.modules.get(modname)
        if net is not None and hasattr(net, "DistributedInstanceNorm2d"):
            net.DistributedInstanceNorm2d = DistributedInstanceNorm2d
