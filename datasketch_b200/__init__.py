"""datasketch_b200 -- a Hopper (H100, sm_90a) MinHash / LSH signature engine that keeps
the API surface of ekzhu/datasketch for the bulk-signature / LSH hot path.

Importing the package loads ``libdsk_b200.so`` (hand-written CUDA behind a C-ABI,
``include/dsk.h``).  There is no CPU fallback: a missing library fails the import,
a missing GPU raises RuntimeError on the first compute call.
"""
from . import _native

_native.load()  # fail loudly if the CUDA library is absent

from .hashfunc import murmur3_hash32, sha1_hash32, sha1_hash64, xxh32_hash32  # noqa: E402
from .minhash import MinHash  # noqa: E402
from .lean_minhash import LeanMinHash  # noqa: E402
from .b_bit_minhash import bBitMinHash  # noqa: E402
from .weighted_minhash import WeightedMinHash, WeightedMinHashGenerator  # noqa: E402
from .lsh import GpuLSH, MinHashLSH, MinHashLSHDeletionSession, MinHashLSHInsertionSession  # noqa: E402
from .lshforest import GpuLSHForest, MinHashLSHForest  # noqa: E402
from .lshensemble import GpuLSHEnsemble, MinHashLSHEnsemble  # noqa: E402
from .lsh_bloom import MinHashLSHBloom  # noqa: E402
from . import codec, distributed, engine, shingle  # noqa: E402

# aliases kept by the reference (datasketch/__init__.py)
WeightedMinHashLSH = MinHashLSH
WeightedMinHashLSHForest = MinHashLSHForest

__version__ = "0.1.0"
__all__ = ["MinHash", "LeanMinHash", "bBitMinHash", "WeightedMinHash", "WeightedMinHashGenerator", "MinHashLSH", "GpuLSH", "MinHashLSHForest", "GpuLSHForest", "MinHashLSHEnsemble", "GpuLSHEnsemble", "MinHashLSHBloom", "MinHashLSHBloom",
           "WeightedMinHashLSH", "WeightedMinHashLSHForest", "MinHashLSHInsertionSession", "MinHashLSHDeletionSession", "sha1_hash32", "sha1_hash64", "xxh32_hash32", "murmur3_hash32", "engine", "codec", "distributed", "shingle"]
