# -*- coding: utf-8 -*-
"""I/O glue mirroring ``wavenet_vocoder/utils/utils.py`` (reference v0.1.1): same function names,
arguments and error behaviour (``logging.error`` + ``sys.exit(1)``), so the CLIs and recipes keep working.

Differences (SURVEY.md section 2 row 8 / 8f.2): ``h5py`` and ``soundfile`` are imported lazily, and every
HDF5 helper also accepts a ``.npz`` file (same dataset paths as keys) so that the data plumbing can be
exercised on hosts without h5py.  None of this is on the GPU hot path.
"""
import fnmatch
import logging
import os
import sys
import threading

import numpy as np


def _h5py():
    try:
        import h5py
        return h5py
    except ImportError:
        logging.error("h5py is required to read .h5 files (use .npz feature files otherwise).")
        sys.exit(1)


def _is_npz(name):
    return name.endswith(".npz")


def _key(path):
    return path.strip("/").replace("/", ".")


def check_hdf5(hdf5_name, hdf5_path):
    """CHECK HDF5 EXISTENCE (reference utils.py:18-36)."""
    if not os.path.exists(hdf5_name):
        return False
    if _is_npz(hdf5_name):
        with np.load(hdf5_name) as f:
            return _key(hdf5_path) in f.files
    with _h5py().File(hdf5_name, "r") as f:
        return hdf5_path in f


def read_hdf5(hdf5_name, hdf5_path):
    """READ HDF5 DATASET (reference utils.py:39-63)."""
    if not os.path.exists(hdf5_name):
        logging.error("there is no such a hdf5 file (%s)." % hdf5_name)
        sys.exit(1)
    if _is_npz(hdf5_name):
        with np.load(hdf5_name) as f:
            if _key(hdf5_path) not in f.files:
                logging.error("there is no such a data in hdf5 file. (%s)" % hdf5_path)
                sys.exit(1)
            return f[_key(hdf5_path)]
    with _h5py().File(hdf5_name, "r") as f:
        if hdf5_path not in f:
            logging.error("there is no such a data in hdf5 file. (%s)" % hdf5_path)
            sys.exit(1)
        return f[hdf5_path][()]


def shape_hdf5(hdf5_name, hdf5_path):
    """GET HDF5 DATASET SHAPE (reference utils.py:66-83)."""
    if not check_hdf5(hdf5_name, hdf5_path):
        logging.error("there is no such a file or dataset")
        sys.exit(1)
    if _is_npz(hdf5_name):
        with np.load(hdf5_name) as f:
            return f[_key(hdf5_path)].shape
    with _h5py().File(hdf5_name, "r") as f:
        return f[hdf5_path].shape


def write_hdf5(hdf5_name, hdf5_path, write_data, is_overwrite=True):
    """WRITE DATASET TO HDF5 (reference utils.py:86-126)."""
    write_data = np.array(write_data)
    folder_name, _ = os.path.split(hdf5_name)
    if not os.path.exists(folder_name) and len(folder_name) != 0:
        os.makedirs(folder_name)
    if _is_npz(hdf5_name):
        data = {}
        if os.path.exists(hdf5_name):
            with np.load(hdf5_name) as f:
                data = {k: f[k] for k in f.files}
        if _key(hdf5_path) in data and not is_overwrite:
            logging.error("dataset in hdf5 file already exists.")
            sys.exit(1)
        data[_key(hdf5_path)] = write_data
        np.savez(hdf5_name, **data)
        return
    h5py = _h5py()
    if os.path.exists(hdf5_name):
        f = h5py.File(hdf5_name, "r+")
        if hdf5_path in f:
            if is_overwrite:
                logging.warning("dataset in hdf5 file already exists.")
                logging.warning("recreate dataset in hdf5.")
                del f[hdf5_path]
            else:
                logging.error("dataset in hdf5 file already exists.")
                logging.error("if you want to overwrite, please set is_overwrite = True.")
                f.close()
                sys.exit(1)
    else:
        f = h5py.File(hdf5_name, "w")
    f.create_dataset(hdf5_path, data=write_data)
    f.flush()
    f.close()


def find_files(directory, pattern="*.wav", use_dir_name=True):
    """FIND FILES RECURSIVELY (reference utils.py:129-147)."""
    files = []
    for root, _, filenames in os.walk(directory, followlinks=True):
        for filename in fnmatch.filter(filenames, pattern):
            files.append(os.path.join(root, filename))
    if not use_dir_name:
        files = [f.replace(directory + "/", "") for f in files]
    return files


def read_txt(file_list):
    """READ TXT FILE (reference utils.py:150-162)."""
    with open(file_list, "r") as f:
        return [line.replace("\n", "") for line in f.readlines()]


class BackgroundGenerator(threading.Thread):
    """Prefetch thread around a generator (reference utils.py:165-205), incl. the py2-style ``next()``."""

    def __init__(self, generator, max_prefetch=1):
        threading.Thread.__init__(self)
        from queue import Queue
        self.queue = Queue(max_prefetch)
        self.generator = generator
        self.daemon = True
        self.start()

    def run(self):
        for item in self.generator:
            self.queue.put(item)
        self.queue.put(None)

    def next(self):
        item = self.queue.get()
        if item is None:
            raise StopIteration
        return item

    def __next__(self):
        return self.next()

    def __iter__(self):
        return self


class background(object):
    """BACKGROUND GENERATOR DECORATOR (reference utils.py:208-217; like there, max_prefetch is not forwarded)."""

    def __init__(self, max_prefetch=1):
        self.max_prefetch = max_prefetch

    def __call__(self, gen):
        def bg_generator(*args, **kwargs):
            return BackgroundGenerator(gen(*args, **kwargs))
        return bg_generator


def extend_time(feats, upsampling_factor):
    """EXTEND TIME RESOLUTION (reference utils.py:220-242): (T, D) -> (upsampling_factor * T, D), float64."""
    return np.repeat(np.asarray(feats, dtype=np.float64), upsampling_factor, axis=0)


# ---- wav I/O: soundfile when present, stdlib `wave` (PCM_16) otherwise -------------------------------------
def read_wav(path, dtype=np.float32):
    """``sf.read(path, dtype=np.float32)`` (reference bin/train.py:121): samples in [-1, 1), sampling rate."""
    try:
        import soundfile as sf
        return sf.read(path, dtype=dtype)
    except ImportError:
        import wave
        with wave.open(path, "rb") as w:
            if w.getsampwidth() != 2 or w.getnchannels() != 1:
                logging.error("without soundfile only mono PCM_16 wav files are supported (%s)." % path)
                sys.exit(1)
            data = np.frombuffer(w.readframes(w.getnframes()), dtype="<i2")
            return (data.astype(dtype) / dtype(32768)), w.getframerate()


def have_soundfile():
    try:
        import soundfile  # noqa: F401
        return True
    except ImportError:
        return False


def write_wav_pcm16(path, pcm, fs):
    """Write int16 samples (already quantised, e.g. by nets.codes_to_pcm16 on the device) as a mono PCM_16 wav."""
    import wave
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(int(fs))
        w.writeframes(np.ascontiguousarray(pcm, dtype="<i2").tobytes())


def read_wav_int16(path):
    """``scipy.io.wavfile.read`` as the reference's feature extraction and noise shaping call it: (fs, samples in the
    file's dtype); the stdlib ``wave`` reader (16-bit PCM) when scipy is missing."""
    try:
        from scipy.io import wavfile
        return wavfile.read(path)
    except ImportError:
        import wave
        with wave.open(path, "rb") as w:
            return w.getframerate(), np.frombuffer(w.readframes(w.getnframes()), dtype="<i2")


def write_wav_int16(path, fs, x):
    """``scipy.io.wavfile.write(path, fs, x)`` of int16 samples; ``write_wav_pcm16`` when scipy is missing."""
    try:
        from scipy.io import wavfile
        wavfile.write(path, fs, x)
    except ImportError:
        write_wav_pcm16(path, x, fs)


def write_wav(path, x, fs):
    """``sf.write(path, x, fs, "PCM_16")`` (reference bin/decode.py:319)."""
    try:
        import soundfile as sf
        sf.write(path, x, fs, "PCM_16")
    except ImportError:
        import wave
        pcm = np.clip(np.round(np.asarray(x, dtype=np.float64) * 32768.0), -32768, 32767).astype("<i2")
        with wave.open(path, "wb") as w:
            w.setnchannels(1)
            w.setsampwidth(2)
            w.setframerate(int(fs))
            w.writeframes(pcm.tobytes())


class WavWriter(object):
    """Mono PCM_16 wav written chunk by chunk, byte-identical to ``write_wav`` (float samples, ``write``) or
    ``write_wav_pcm16`` (int16 samples, ``write_pcm16``) of the whole signal: soundfile's ``SoundFile`` in write mode when
    present, else the stdlib ``wave`` writer; both patch the RIFF sizes on ``close``."""

    def __init__(self, path, fs):
        try:
            import soundfile as sf
            self._sf = sf.SoundFile(path, "w", int(fs), 1, "PCM_16")
            self._w = None
        except ImportError:
            import wave
            self._sf = None
            self._w = wave.open(path, "wb")
            self._w.setnchannels(1)
            self._w.setsampwidth(2)
            self._w.setframerate(int(fs))

    def write(self, x):
        if self._sf is not None:
            self._sf.write(np.asarray(x))
        else:
            self.write_pcm16(np.clip(np.round(np.asarray(x, dtype=np.float64) * 32768.0), -32768, 32767))

    def write_pcm16(self, pcm):
        if self._sf is not None:
            self._sf.write(np.ascontiguousarray(pcm, dtype=np.int16))
        else:
            self._w.writeframes(np.ascontiguousarray(pcm, dtype="<i2").tobytes())

    def close(self):
        (self._sf if self._sf is not None else self._w).close()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()
