// The generic quasiseparable scans for state dimension J = 4 (see qs_generic.cuh): a translation unit of its own so that
// it compiles in parallel with quasisep.cu.
#include "qs_generic.cuh"

QS_FOR_J(template, 4)
