#pragma once
#include "ref_ros.h"
