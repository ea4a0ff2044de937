"""loexec — H100-native executor for learningOrchestra's projection -> type-cast -> histogram path.

Layout (DESIGN.md):
  csrc/            sm_90a kernels + the C ABI of include/loexec.h  ->  lib/libloexec.so
  _native, engine  ctypes binding and the Engine / DeviceTable object layer
  projection, data_type_update, histogram, utils, server
                   drop-in mirrors of the reference's service classes and REST routes
  columnar         documents <-> columns adapter;  table_cache: datasets resident in HBM
  column_store     the wrapper API over rows stored as columns (Arrow text / float64), CSV ingest
  sharding         ShardedEngine: several GPUs behind the Engine methods (lo_group_* in the library)

There is no CPU fallback: without libloexec.so and an H100 every compute entry raises LoexecError.
"""
__version__ = "0.1.0"
