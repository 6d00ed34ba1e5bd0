"""chattts_b200 - H100-native (sm_90a) hot paths of ChatTTS behind the reference's API.

    from chattts_b200 import Chat          # same surface as ChatTTS.Chat (core.py)

Importing the package never touches CUDA; the kernels live in ``lib/libchattts_b200.so``
(``python -m chattts_b200.build``) and every product call fails loudly without it / without a GPU.
"""
from .config import Config  # noqa: F401

__all__ = ["Chat", "Config"]


def __getattr__(name):
    if name == "Chat":
        from .core import Chat

        return Chat
    raise AttributeError(name)
