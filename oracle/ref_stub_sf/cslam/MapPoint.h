// see KeyFrame.h in this directory
#include <cslam/KeyFrame.h>
