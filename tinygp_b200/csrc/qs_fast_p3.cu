// Layout-specialised quasiseparable kernels of the layouts 13, 21, 37 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(13) X(21) X(37)
#include "qs_fast.cu"
