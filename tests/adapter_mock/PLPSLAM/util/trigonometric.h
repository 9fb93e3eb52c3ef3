#pragma once
namespace PLPSLAM { namespace util { float cos(float v); } }  // util/trigonometric.h: the polynomial cosine
