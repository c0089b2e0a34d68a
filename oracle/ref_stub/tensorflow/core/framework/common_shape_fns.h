#include "tf_stub.h"
