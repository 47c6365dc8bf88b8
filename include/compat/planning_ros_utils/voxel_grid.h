/* forwards the reference header name to the host layer of libmplb (see INTEGRATION.md section 3.1) */
#pragma once
#include <mpl_b200/voxel_grid.hpp>
