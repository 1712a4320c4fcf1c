from .utils import *  # noqa
from .utils import have_soundfile, read_wav, write_wav, write_wav_pcm16, WavWriter  # noqa
from .utils import read_wav_int16, write_wav_int16  # noqa
