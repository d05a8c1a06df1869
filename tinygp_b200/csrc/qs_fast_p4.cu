// Layout-specialised quasiseparable kernels of the layouts 25, 22, 85 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(25) X(22) X(85)
#include "qs_fast.cu"
