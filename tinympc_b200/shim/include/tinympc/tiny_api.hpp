// forwarding header: the reference layout <tinympc/tiny_api.hpp> -> the H100 shim
#pragma once
#include "../../tinympc_shim.hpp"
