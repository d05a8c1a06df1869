// Layout-specialised quasiseparable kernels of the layouts 1, 2, 3, 5 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(1) X(2) X(3) X(5)
#include "qs_fast.cu"
