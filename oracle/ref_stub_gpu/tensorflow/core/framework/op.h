#include "../../../tf_gpu_stub.h"
