#pragma once
#include "ref_ceres.h"
