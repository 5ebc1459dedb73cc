// see MapPoint.h in this directory
#include <cslam/MapPoint.h>
