// Drop-in for the reference header of the same path; everything lives in hexl/b200/hexl_api.hpp.
#pragma once
#include "../../b200/hexl_api.hpp"
