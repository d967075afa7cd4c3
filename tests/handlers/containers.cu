// The container script handler's entry points: compiled to an sm_90a cubin by beta9_b200.build.build_test_handlers
// (build() makes tests/handlers/containers.cubin) for tests/test_gpu_user_containers.py.
#include "containers.cuh"

B9_HANDLER(cscript, b9_containers::CScript)
