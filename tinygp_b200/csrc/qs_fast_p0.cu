// Layout-specialised quasiseparable kernels of the layout 10 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(10)
#include "qs_fast.cu"
