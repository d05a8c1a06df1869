// Layout-specialised quasiseparable kernels of the layout 14 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(14)
#include "qs_fast.cu"
