#pragma once
#include "../core/core.hpp"
