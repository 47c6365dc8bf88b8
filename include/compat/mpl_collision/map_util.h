/* forwards the reference header name to the host layer of libmplb (see INTEGRATION.md section 2) */
#pragma once
#include <mpl_b200/map_planner.hpp>
