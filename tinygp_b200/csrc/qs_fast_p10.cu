// Layout-specialised quasiseparable kernels of the layout 41 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(41)
#include "qs_fast.cu"
