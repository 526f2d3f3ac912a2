// ORACLE — TEST INFRASTRUCTURE ONLY. Stand-in for <ros/package.h> (globalmap_gene.cpp's PCD path, never taken).
#pragma once
#include <string>
namespace ros { namespace package { inline std::string getPath(const std::string &) { return std::string(); } } }
