// see Frame.h in this directory
#include <cslam/Frame.h>
