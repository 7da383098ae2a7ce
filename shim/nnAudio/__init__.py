"""Import shim: put ``<repo>/shim`` (and ``<repo>``) on ``sys.path`` and existing code that
does ``from nnAudio import features`` / ``from nnAudio.Spectrogram import STFT`` runs on the
H100-native engine unchanged (mirrors nnAudio/__init__.py:1)."""
__version__ = "0.3.3+nnaudio_b200"
