// Layout-specialised quasiseparable kernels of the layouts 6, 9, 7 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(6) X(9) X(7)
#include "qs_fast.cu"
