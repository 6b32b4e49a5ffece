//go:build cuda && cgo

// Drop-in file for github.com/cloudflare/circl/sign/schemes (next to schemes.go): with the `cuda` build tag "Ed25519",
// "Ed448", "Ed25519-Dilithium2", "Ed448-Dilithium3" and "ML-DSA-65" (sign/schemes/schemes.go:31-54) are served by the
// cb200 engine, in their places of allSchemes; ByName (schemes.go:56-71) is unchanged.
//
// Delivered as source: the build image has no Go toolchain (see INTEGRATION.md section 3).
package schemes

import (
	"strings"

	"github.com/cloudflare/circl/sign"

	"example.com/circl_b200/go/cb200"
	"example.com/circl_b200/go/ed25519cuda"
	"example.com/circl_b200/go/ed448cuda"
	"example.com/circl_b200/go/eddilithium2cuda"
	"example.com/circl_b200/go/eddilithium3cuda"
	"example.com/circl_b200/go/mldsa65cuda"
)

// The file name sorts after schemes.go on purpose: the init functions of a package run in file-name order and the map
// written here is made by the init of schemes.go.
func init() {
	if cb200.Init() != nil {
		return
	}
	for _, s := range []sign.Scheme{ed25519cuda.Scheme(), ed448cuda.Scheme(), eddilithium2cuda.Scheme(),
		eddilithium3cuda.Scheme(), mldsa65cuda.Scheme()} {
		name := strings.ToLower(s.Name())
		allSchemeNames[name] = s
		for i := range allSchemes {
			if strings.ToLower(allSchemes[i].Name()) == name {
				allSchemes[i] = s
			}
		}
	}
}
