"""`densephrases`: import-compatible facade of princeton-nlp/DensePhrases' package (densephrases/__init__.py:1-4) over
densephrases_b200, so `from densephrases import MIPS, Encoder, Options, DensePhrases` and the `densephrases.utils.*`
imports of eval_phrase_retrieval.py:19-25 resolve to the H100-native implementation."""
from densephrases_b200.encoder import Encoder  # noqa: F401
from densephrases_b200.mips import MIPS, MIPSIndex  # noqa: F401
from densephrases_b200.options import Options  # noqa: F401
from densephrases_b200.runtime import DensePhrases  # noqa: F401
