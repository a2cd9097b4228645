#pragma once
#include "srl_lk_cv.h"
