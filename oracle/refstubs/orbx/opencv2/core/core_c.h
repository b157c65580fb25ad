#pragma once
#include "core.hpp"
