"""Drop-in alias: ``import wavenet_vocoder`` resolves to the H100 build (pytorchwavenetvocoder_b200), so the
reference's recipes (``egs/*/run.sh`` call ``wavenet_vocoder/bin/{train,decode}.py`` by name) and user code
(``from wavenet_vocoder.nets import WaveNet``) run unchanged."""
__version__ = "0.1.1+b200"
