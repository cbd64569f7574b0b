"""Data side of the hot path with the reference's names (reference audio_data.py).

* ``mu_law_encoding`` / ``mu_law_expansion`` / ``quantize_data``  (audio_data.py:133-158; note mu = classes, not classes - 1)
* ``WavenetDataset``  the reference's item arithmetic over a ``dataset.npz`` of quantised uint8 audio (audio_data.py:12-131)
  with one addition (SURVEY.md section 8, row f2): ``one_hot=False`` makes ``__getitem__`` return the ``item_length`` class
  INDICES (uint8) instead of a (classes, item_length) float one-hot matrix.  ``WaveNetModel.forward_indices`` gathers the
  start_conv column of each index on the GPU, which is bit-identical to the dense convolution on the one-hot input and
  moves 1 byte per sample over PCIe / HBM instead of 1 KB.
* ``condition_on_file=True`` makes items ``(x, file_index, target)``: the index of the array that holds the item's last
  target sample, a class label for training a model conditioned on the file (``WaveNetModel(condition_channels=...)``).
* ``write_wav``  16-bit PCM writer for generated audio (the reference calls librosa.output.write_wav, generate_script.py:35;
  librosa is not a dependency here).
Building a dataset from audio files (``create_dataset``) needs librosa exactly as in the reference and raises without it.
"""
import bisect
import math
import os
import wave

import numpy as np
import torch
import torch.utils.data


def mu_law_encoding(data, mu):
    return np.sign(data) * np.log(1 + mu * np.abs(data)) / np.log(mu + 1)


def mu_law_expansion(data, mu):
    return np.sign(data) * (np.exp(np.abs(data) * np.log(mu + 1)) - 1) / mu


def quantize_data(data, classes):
    mu_x = mu_law_encoding(data, classes)
    bins = np.linspace(-1, 1, classes)
    return np.digitize(mu_x, bins) - 1


def list_all_audio_files(location):
    found = []
    for dirpath, _, names in os.walk(location):
        found += [os.path.join(dirpath, n) for n in names if n.lower().endswith((".mp3", ".wav", ".aif", ".aiff"))]
    if not found:
        print("found no audio files in " + location)
    return found


def write_wav(path, audio, sr=16000):
    """float waveform in [-1, 1] -> mono 16-bit PCM .wav (what generate_script.py:35 does through librosa)."""
    pcm = np.clip(np.asarray(audio, dtype=np.float64), -1.0, 1.0)
    pcm = np.round(pcm * 32767.0).astype("<i2")
    with wave.open(path, "wb") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(int(sr))
        f.writeframes(pcm.tobytes())


class WavenetDataset(torch.utils.data.Dataset):
    """Items of ``item_length`` input samples and the ``target_length`` samples that follow, cut from the concatenation of
    the arrays in ``dataset_file`` (``arr_0``, ``arr_1``, ...); every ``test_stride``-th item belongs to the test split
    (reference audio_data.py:12-131: same item index -> sample offset map, same cross-file reads)."""

    def __init__(self, dataset_file, item_length, target_length, file_location=None, classes=256, sampling_rate=16000,
                 mono=True, normalize=False, dtype=np.uint8, train=True, test_stride=100, one_hot=True,
                 condition_on_file=False):
        self.dataset_file = dataset_file
        self._item_length = item_length
        self._test_stride = test_stride
        self.target_length = target_length
        self.classes = classes
        self.one_hot = one_hot
        self.condition_on_file = condition_on_file
        self.mono = self.normalize = self.sampling_rate = self.dtype = None      # unknown for an existing file, as upstream
        if not os.path.isfile(dataset_file):
            assert file_location is not None, "no location for dataset files specified"
            self.mono, self.normalize, self.sampling_rate, self.dtype = mono, normalize, sampling_rate, dtype
            self.create_dataset(file_location, dataset_file)
        self.data = np.load(self.dataset_file, mmap_mode='r')
        self.start_samples = [0]
        self._length = 0
        self.calculate_length()
        self.train = train

    def create_dataset(self, location, out_file):
        try:
            import librosa as lr
        except ImportError as e:
            raise RuntimeError("building a dataset from audio files needs librosa (as in the reference); "
                               "an existing dataset.npz does not") from e
        print("create dataset from audio files at", location)
        self.dataset_file = out_file
        arrays = []
        for i, name in enumerate(list_all_audio_files(location)):
            audio, _ = lr.load(path=name, sr=self.sampling_rate, mono=self.mono)
            if self.normalize:
                audio = lr.util.normalize(audio)
            arrays.append(quantize_data(audio, self.classes).astype(self.dtype))
        np.savez(self.dataset_file, *arrays)

    def calculate_length(self):
        starts = [0]
        for i in range(len(self.data.keys())):
            starts.append(starts[-1] + len(self.data['arr_' + str(i)]))
        available = starts[-1] - (self._item_length - (self.target_length - 1)) - 1
        self._length = math.floor(available / self.target_length)
        self.start_samples = starts

    def set_item_length(self, l):
        self._item_length = l
        self.calculate_length()

    def _sample_index(self, idx):
        if self._test_stride < 2:
            return idx * self.target_length
        if self.train:
            return idx * self.target_length + math.floor(idx / (self._test_stride - 1))
        return self._test_stride * (idx + 1) - 1

    def _read(self, start, n):
        """n consecutive samples of the concatenated arrays starting at `start` (at most two arrays, as upstream)."""
        fi = max(bisect.bisect_left(self.start_samples, start) - 1, 0)
        pos = start - self.start_samples[fi]
        spill = start + n - self.start_samples[fi + 1]
        first = self.data['arr_' + str(fi)]
        if spill < 0:
            return np.asarray(first[pos:pos + n])
        return np.concatenate((np.asarray(first[pos:]), np.asarray(self.data['arr_' + str(fi + 1)][:spill])))

    def file_index(self, idx):
        """Index of the array that holds the last target sample of item ``idx``."""
        return bisect.bisect_right(self.start_samples, self._sample_index(idx) + self._item_length) - 1

    def __getitem__(self, idx):
        sample = self._read(self._sample_index(idx), self._item_length + 1)
        target = torch.from_numpy(sample[-self.target_length:].astype(np.int64)).unsqueeze(0)
        if not self.one_hot:
            x = torch.from_numpy(sample[:self._item_length].astype(np.uint8))
        else:
            example = torch.from_numpy(sample[:self._item_length].astype(np.int64))
            x = torch.zeros(self.classes, self._item_length)
            x.scatter_(0, example.unsqueeze(0), 1.)
        if self.condition_on_file:
            return x, torch.tensor(self.file_index(idx), dtype=torch.int64), target
        return x, target

    def __len__(self):
        test_length = math.floor(self._length / self._test_stride)
        return self._length - test_length if self.train else test_length
