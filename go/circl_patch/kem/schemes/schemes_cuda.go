//go:build cuda && cgo

// Drop-in file for github.com/cloudflare/circl/kem/schemes (next to schemes.go): with the `cuda` build tag the registry
// entries "ML-KEM-768", "ML-KEM-1024", "X-Wing", "HPKE_KEM_X25519_HKDF_SHA256", "HPKE_KEM_X448_HKDF_SHA512",
// "HPKE_KEM_P256_HKDF_SHA256", "HPKE_KEM_P384_HKDF_SHA384", "HPKE_KEM_P521_HKDF_SHA512" and "FrodoKEM-640-SHAKE"
// (kem/schemes/schemes.go:30-55) are served by the cb200 engine; every
// other scheme, and every build without the tag, is untouched.  ByName keeps matching on the lower-cased Name()
// (schemes.go:57-72), which the GPU schemes do not change.
//
// Delivered as source: the build image has no Go toolchain (see INTEGRATION.md section 3).
package schemes

import (
	"strings"

	"github.com/cloudflare/circl/kem"

	"example.com/circl_b200/go/cb200"
	"example.com/circl_b200/go/frodo640shakecuda"
	"example.com/circl_b200/go/hpkecuda"
	"example.com/circl_b200/go/mlkem1024cuda"
	"example.com/circl_b200/go/mlkem768cuda"
	"example.com/circl_b200/go/xwingcuda"
)

// The file name sorts after schemes.go on purpose: the init functions of a package run in file-name order and the map
// written here is made by the init of schemes.go.
func init() {
	if cb200.Init() != nil { // no usable H100: keep CIRCL's own schemes (the library itself has no CPU fallback)
		return
	}
	for _, s := range []kem.Scheme{mlkem768cuda.Scheme(), mlkem1024cuda.Scheme(), xwingcuda.Scheme(), hpkecuda.X25519(),
		hpkecuda.X448(), hpkecuda.P256(), hpkecuda.P384(), hpkecuda.P521(), frodo640shakecuda.Scheme()} {
		name := strings.ToLower(s.Name())
		allSchemeNames[name] = s
		for i := range allSchemes {
			if strings.ToLower(allSchemes[i].Name()) == name {
				allSchemes[i] = s
			}
		}
	}
}
