// Layout-specialised quasiseparable kernels of the layout 42 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(42)
#include "qs_fast.cu"
