"""speecht5_b200 -- H100-native (sm_90a) implementation of the SpeechT5 data-parallel forward/backward hot path behind
the reference's fairseq plugin surface (`--user-dir speecht5_b200`: task "speecht5", criterion "speecht5", model
"t5_transformer" + arch presets), cf. /root/reference/SpeechT5/speecht5/__init__.py:1."""
from . import criterions, models, tasks  # noqa: F401
from .ops import RT  # noqa: F401
