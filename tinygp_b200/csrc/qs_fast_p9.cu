// Layout-specialised quasiseparable kernels of the layout 26 (see qs_fast.cu).
#define QSF_PART_LAYOUTS(X) X(26)
#include "qs_fast.cu"
