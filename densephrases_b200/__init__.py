"""densephrases_b200: H100-native (sm_90a) implementation of the DensePhrases retrieval hot path
(query encoder forward + IVF-PQ maximum-inner-product search), see DESIGN.md."""
from .ivfpq import IndexFilter, IvfPqIndex, QueryFilters, merge_shards  # noqa: F401
