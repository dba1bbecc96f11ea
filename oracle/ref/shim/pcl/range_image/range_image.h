#pragma once
#include "ref_pcl.h"
