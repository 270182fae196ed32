// forwarding header: the reference layout <tinympc/types.hpp> -> the H100 shim
#pragma once
#include "../../tinympc_shim.hpp"
