"""Drop-in for the reference's ``whenet.py``: ``from whenet import WHENet`` keeps working
(reference demo.py:3, demo_video.py:6); the class is the H100-native one."""
from whenet_b200 import WHENet  # noqa: F401
