"""dcb200: H100-native (sm_90a) inference engine for the DeepConsensus hot path.

Scope: `quick_inference.run_model_on_examples` ->
`EncoderOnlyLearnedValuesTransformer` forward -> argmax/QV -> `stitch_utils`
output surface.  The compute path is hand-written CUDA behind a C-ABI
(`include/dcb200.h`, built into `deepconsensus_b200/csrc/libdcb200.so`); this
package is the Python host side that mirrors the reference's interfaces for
that path.  Nothing in this package imports `oracle/` (test infrastructure).
"""

__version__ = "0.1.0"

from deepconsensus_b200 import constants  # noqa: F401
