# -*- coding: utf-8 -*-
"""pytorchwavenetvocoder_b200 -- H100 (sm_90a) native WaveNet vocoder hot paths.

Drop-in for the two hot paths of kan-bayashi/PytorchWaveNetVocoder (training forward/backward through
the residual stack, autoregressive fast generation) behind the reference's own module surface
(``pytorchwavenetvocoder_b200.nets`` mirrors ``wavenet_vocoder.nets``).  All device arithmetic is in
``libwnb200.so`` (hand-written CUDA, C ABI in ``include/wnb200.h``); see DESIGN.md.
"""
__version__ = "0.1.0"
