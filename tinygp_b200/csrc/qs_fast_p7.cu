// Layout-specialised quasiseparable kernels of the layout 11 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(11)
#include "qs_fast.cu"
