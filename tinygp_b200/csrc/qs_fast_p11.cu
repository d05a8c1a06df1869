// Layout-specialised quasiseparable kernels of the layout 38 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(38)
#include "qs_fast.cu"
