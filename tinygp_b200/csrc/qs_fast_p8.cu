// Layout-specialised quasiseparable kernels of the layout 15 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(15)
#include "qs_fast.cu"
