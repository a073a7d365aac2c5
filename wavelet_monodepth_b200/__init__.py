"""H100-native (sm_90a) implementation of the wavelet-monodepth decoder hot path.

Public surface = the reference's (nianticlabs/wavelet-monodepth) own API for this path:

  wavelets       DWTForward / DWTInverse (aliases DWT / IDWT)      <- pytorch_wavelets
  kitti_layers   ConvBlock, Conv3x3, Conv1x1, upsample, sparse_*   <- KITTI/layers.py
  kitti_decoders DepthDecoder, DepthWaveProgressiveDecoder,
                 SparseDepthWaveProgressiveDecoder                 <- KITTI/networks/decoders/depth_decoder.py
  nyu_decoders   Conv3x3, UpSampleBlock, DecoderWave,
                 SparseDecoderWave                                 <- NYUv2/networks/{layers,decoders/densedepth_decoder}.py
  nyu_loss       NyuDepthLoss: the NYUv2 training objective,
                 forward and backward, deterministic               <- NYUv2/train.py:279-327
  kitti_loss     KittiDepthHintsLoss: KITTI's stereo depth-hints
                 objective, forward and backward, deterministic    <- KITTI/trainer.py:329-560
  shard          batch sharding + the single all-gather (one process per GPU)
  ops / _lib     tensor-level wrappers over the C ABI of libwmd.so (include/wmd.h)

Importing the package does not load the CUDA library; the first op does, and raises if it is missing.
There is no CPU fallback.
"""
from . import synth, opcount  # noqa: F401  (host-only helpers)

__all__ = ["wavelets", "kitti_layers", "kitti_decoders", "nyu_decoders", "shard", "ops", "synth", "opcount"]
