"""`simuleval --agent <this file>`: the H100-engine drop-in for the reference's agent/speech_to_text.wait-k-stride-n.agent.py (UnitY checkpoints).

SimulEval imports the file as a top-level module and expects exactly ONE @entrypoint class in it
(SimulEval/simuleval/utils/agent.py:25-56); the implementation lives in streamspeech_b200/waitk.py."""
import os
import sys

_REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
if _REPO not in sys.path:
    sys.path.insert(0, _REPO)

from streamspeech_b200 import waitk as _impl  # noqa: E402
from streamspeech_b200.simuleval_compat import entrypoint  # noqa: E402


@entrypoint
class WaitkS2TTAgent(_impl.WaitkS2TTAgent):
    pass
