// The contract handlers' entry points: compiled to an sm_90a cubin by beta9_b200.build.build_test_handlers (build()
// makes tests/handlers/contract.cubin) for tests/test_gpu_handler_contract.py.
#include "contract.cuh"

B9_HANDLER(script, b9_contract::Script)
B9_HANDLER(script_sig, b9_contract::ScriptSig)
B9_HANDLER(inspect, b9_contract::Inspect)
B9_HANDLER(inspect_keys, b9_contract::InspectKeys)
